"""Step time of the fused self-critical step under each sampler setting and table kind, per family at recipe size: the default
(multinomial samples, greedy baseline, pickle document frequencies) against top-k / nucleus / greedy train samples, sampled baselines and
a corpus table (init_scorer('corpus'): document frequencies rebuilt on the device every step).  10 images x 5 samples, 36 regions, V = 9487,
T = 16; UpDown E = H = 1000, A = 512 (configs/updown); Att2in2 and NewFC E = H = A = 512; AoANet E = H = 1024, 8 heads (configs/aoa.yml);
Transformer 6 + 6 layers, d_model 512, d_ff 2048, 8 heads.  Each setting is warmed up through its eager step, its capture and a replay, so
the windows time graph replays, as training does.  Prints one JSON line with the card name and power limit read in the same run.

    python tools/scst_sampler_rate.py [--steps 10] [--warmup 3] [--repeats 5] [--families updown,aoa]
"""
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

BASE = dict(V=9487, F_fc=2048, F_att=2048, T=16)
DIMS = {'updown': dict(BASE, E=1000, H=1000, A=512), 'att2in2': dict(BASE, E=512, H=512, A=512), 'newfc': dict(BASE, E=512, H=512, A=512),
        'aoa': dict(BASE, E=1024, H=1024, A=0), 'transformer': dict(BASE, E=512, H=2048, A=6)}
SETTINGS = {'default': {}, 'train_top5': dict(sample_method='top5'), 'train_top0.9': dict(sample_method='top0.9'),
            'train_greedy': dict(sample_method='greedy'), 'baseline_sample': dict(baseline_method='sample'),
            'baseline_top0.9': dict(baseline_method='top0.9'), 'corpus_table': {}}


def timed(step, steps, warmup, repeats):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    ms = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        for _ in range(steps):
            step()
        torch.cuda.synchronize()
        ms.append(1e3 * (time.perf_counter() - t0) / steps)
    return {'ms_per_step': round(statistics.median(ms), 3), 'ms_min': round(min(ms), 3), 'ms_max': round(max(ms), 3)}


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--steps', type=int, default=10)
    p.add_argument('--warmup', type=int, default=3)
    p.add_argument('--repeats', type=int, default=5)
    p.add_argument('--mode', default='tc_f16x3', choices=['tc_f16x3', 'simt_fp32'])
    p.add_argument('--families', default='updown,att2in2,newfc,aoa,transformer')
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('scst_sampler_rate.py measures on a CUDA device; none is visible')
    from imagecaptioning.pytorch_b200 import rewards
    from imagecaptioning.pytorch_b200 import synthetic as syn
    B, n, R = 10, 5, 36
    out = {'images': B, 'per_image': n, 'regions': R, 'mode': a.mode, 'steps_per_window': a.steps, 'windows': a.repeats}
    for family in a.families.split(','):
        cfg = DIMS[family]
        model = syn.build_model(family, seed=1234, logit_scale=6.0, mode=a.mode, device=torch.device('cuda:0'), heads=8, **cfg)
        model.train()
        fc, att = syn.make_inputs(B, R, cfg['F_fc'], cfg['F_att'], seed=1234)
        fc, att = fc.cuda(), att.cuda()
        if family == 'newfc':
            att = fc.new_zeros(B, 0, 0)
        refs = syn.make_refs(200, cfg['V'], seed=4)
        tables = {'pickle': rewards.CiderDTable(*syn.document_frequency(refs)), 'corpus': rewards.CorpusCiderDTable()}
        gts = refs[:B]
        res = {'dims': cfg}
        for name, kw in SETTINGS.items():
            table = tables['corpus' if name == 'corpus_table' else 'pickle']
            res[name] = timed(lambda: model.scst_step(fc, att, gts, table, n, **kw), a.steps, max(3, a.warmup), a.repeats)
        for name in SETTINGS:
            if name != 'default':
                res[name]['over_default'] = round(res[name]['ms_per_step'] / res['default']['ms_per_step'], 3)
        out[family] = res
        del model
        torch.cuda.empty_cache()
    out.update(device_info())
    print(json.dumps(out))


if __name__ == '__main__':
    main()
