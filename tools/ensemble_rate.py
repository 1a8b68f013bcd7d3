"""Cost of a test-time ensemble: beam search of K = 1, 2 and 3 UpDown members at BASELINE.json configs[1] dimensions (V 9487, E = H = 1000,
A 512, 36 regions of 2048 features, T 20), batch 256, beam 5, against the single model alone.

    python tools/ensemble_rate.py [--batch 256] [--beam 5] [--rounds 5] [--warmup 2] [--mode tc_f16x3]

Every configuration runs on a side stream, where the beam loop is captured into a CUDA graph and replayed.  After the warm-up the
configurations are timed in alternation, one decode each per round (host clock around work that ends in a device synchronise), and the
median per configuration is reported.  The mixing pass reads K * rows * (V+1) * 4 bytes of member logits per step, twice (statistics pass,
mixing pass).  Prints one JSON line with the device name and power limit beside the numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tools'))

from dbs_rate import device_info      # noqa: E402


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--batch', type=int, default=256)
    p.add_argument('--beam', type=int, default=5)
    p.add_argument('--rounds', type=int, default=5)
    p.add_argument('--warmup', type=int, default=2)
    p.add_argument('--mode', default='tc_f16x3', choices=['tc_f16x3', 'tc_f16x1', 'simt_fp32'])
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('ensemble_rate.py measures on a CUDA device; none is visible')
    import imagecaptioning.pytorch_b200 as b200
    from imagecaptioning.pytorch_b200 import synthetic as syn
    cfg = dict(V=9487, E=1000, H=1000, A=512, F_fc=2048, F_att=2048, T=20)
    dev = torch.device('cuda:0')
    members = [syn.build_model('updown', seed=1234 + k, logit_scale=12.0, mode=a.mode, device=dev, **cfg) for k in range(3)]
    runs = {'single': members[0]}
    for K in (1, 2, 3):
        runs['ensemble_k%d' % K] = b200.B200AttEnsemble(members[:K])
    fc, att = syn.make_inputs(a.batch, 36, cfg['F_fc'], cfg['F_att'], seed=1234)
    fc, att = fc.cuda(), att.cuda()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    opt = {'beam_size': a.beam, 'sample_n': 1}
    times = {name: [] for name in runs}
    launches = {}
    with torch.no_grad(), torch.cuda.stream(side):
        for name, model in runs.items():
            for _ in range(a.warmup):
                model(fc, att, None, opt=opt, mode='sample')
        torch.cuda.synchronize()
        for _ in range(a.rounds):
            for name, model in runs.items():
                l0 = model.launch_count
                t0 = time.perf_counter()
                model(fc, att, None, opt=opt, mode='sample')
                torch.cuda.synchronize()
                times[name].append(time.perf_counter() - t0)
                launches[name] = model.launch_count - l0
    rows, V1 = a.batch * a.beam, cfg['V'] + 1
    out = {'workload': 'UpDown beam %d, batch %d, T %d, V %d, H %d, 36x2048 regions, %s' % (a.beam, a.batch, cfg['T'], cfg['V'], cfg['H'], a.mode),
           'device': device_info(), 'rounds': a.rounds}
    for name, ts in times.items():
        ms = 1e3 * statistics.median(ts)
        out[name] = {'ms_per_decode': round(ms, 3), 'captions_per_s': round(a.batch / (ms / 1e3), 1), 'spread_ms': round(1e3 * (max(ts) - min(ts)), 3),
                     'launches_per_decode': launches[name]}
        if name.startswith('ensemble'):
            K = int(name[-1])
            out[name]['vs_single'] = round(ms / out['single']['ms_per_decode'], 3)
            out[name]['mix_logit_bytes_per_step'] = K * rows * V1 * 4
    print(json.dumps(out))


if __name__ == '__main__':
    main()
