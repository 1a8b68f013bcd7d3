"""Throughput of NewFC's fused training steps at the fc recipe dimensions (configs/fc*.yml with the opts defaults: E = H = 512, F_fc = 2048,
V = 9487, T = 20, labels of 16 + 2 columns, 10 images per batch, 5 captions / samples per image).

    python tools/newfc_rate.py [--steps 20] [--warmup 3] [--repeats 5] [--mode tc_f16x3]

Three measurements on synthetic, seeded, device-resident inputs (att_feats [B, 0, 0], as the reference loader hands NewFC), each a window of
--steps calls ending in a device synchronise, repeated --repeats times to show the spread:
* xe:  the fused XE step (fc.yml) with scheduled sampling at ss_prob 0.25 and dropout 0.5;
* sc:  the fused SCST step (fc_rl.yml) with the greedy baseline, replayed from its step graph after the eager and capturing calls;
* nsc: the 'new_self_critical' step (fc_nsc.yml, leave-one-out baseline), replayed from its step graph likewise.
Prints one JSON line with ms/step (median, min, max over the windows), samples/s (median), engine launches per step and the device name and
power limit they were measured at.
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


def timed(model, step, rows, steps, warmup, repeats):
    for i in range(warmup):
        step(i)
    torch.cuda.synchronize()
    ms = []
    l0 = model.launch_count
    for r in range(repeats):
        t0 = time.perf_counter()
        for i in range(steps):
            step(1000 + r * steps + i)
        torch.cuda.synchronize()
        ms.append(1e3 * (time.perf_counter() - t0) / steps)
    med = statistics.median(ms)
    return {'ms_per_step': round(med, 3), 'ms_min': round(min(ms), 3), 'ms_max': round(max(ms), 3), 'samples_per_s': round(rows / med * 1e3, 1),
            'launches_per_step': (model.launch_count - l0) / (steps * repeats)}


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--steps', type=int, default=20)
    p.add_argument('--warmup', type=int, default=3)
    p.add_argument('--repeats', type=int, default=5)
    p.add_argument('--mode', default='tc_f16x3', choices=['tc_f16x3', 'tc_f16x1', 'simt_fp32'])
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('newfc_rate.py measures on a CUDA device; none is visible')
    from imagecaptioning.pytorch_b200 import synthetic as syn
    from imagecaptioning.pytorch_b200 import rewards
    cfg = dict(V=9487, E=512, H=512, A=512, F_fc=2048, F_att=2048, T=20)
    B, n, L = 10, 5, 16 + 2
    model = syn.build_model('newfc', seed=1234, logit_scale=12.0, mode=a.mode, device=torch.device('cuda:0'), **cfg)
    fc, _ = syn.make_inputs(B, 1, cfg['F_fc'], cfg['F_att'], seed=1234)
    fc = fc.cuda()
    att = fc.new_zeros(B, 0, 0)
    refs = syn.make_refs(200, cfg['V'], seed=4)
    table = rewards.CiderDTable(*syn.document_frequency(refs))
    gts = refs[:B]
    g = torch.Generator().manual_seed(12)
    labels = torch.zeros(B, n, L, dtype=torch.long)
    masks = torch.zeros(B, n, L)
    for i in range(B):
        for j in range(n):
            k = int(torch.randint(6, L - 1, (1,), generator=g))
            labels[i, j, 1:1 + k] = torch.randint(1, cfg['V'] + 1, (k,), generator=g)
            masks[i, j, :k + 2] = 1
    labels, masks = labels.cuda(), masks.cuda()
    model.train()
    out = {'model': 'newfc', 'dims': 'fc recipe (E=H=512, F_fc=2048, V=9487, T=20, labels 16+2)', 'mode': a.mode, 'images': B, 'per_image': n,
           'steps_per_window': a.steps, 'windows': a.repeats}
    model.ss_prob = 0.25
    out['xe'] = timed(model, lambda s: model.xe_step(fc, att, labels, masks, drop_prob=0.5, seed=s), B * n, a.steps, a.warmup, a.repeats)
    model.ss_prob = 0.0
    out['xe']['ss_prob'] = 0.25
    for name, baseline in (('sc', 'greedy'), ('nsc', 'leave_one_out')):
        out[name] = timed(model, lambda s: model.scst_step(fc, att, gts, table, n, drop_prob=0.5, seed=s, baseline=baseline), B * n, a.steps,
                          max(a.warmup, 3), a.repeats)          # >= 3 warm-up calls: eager, capture, first replay
    out.update(device_info())
    print(json.dumps(out))


if __name__ == '__main__':
    main()
