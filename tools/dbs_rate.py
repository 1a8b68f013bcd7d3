"""Captions/s of diverse beam search against the plain beam search of the same total width, UpDown at BASELINE.json configs[1] dimensions.

    python tools/dbs_rate.py [--batch 256] [--beam 9] [--groups 3] [--steps 10] [--warmup 3] [--rounds 3] [--mode tc_f16x3]

Inputs are synthetic, seeded and device-resident; the timed window holds only decode calls and ends in a device synchronise.  The two
arms alternate within each round so drift on a shared host hits both.  The decode calls run on a side stream, where the engine captures
each beam loop into a CUDA graph (torch's legacy default stream cannot be captured).  The engine keeps one captured loop, so each arm
makes two untimed calls (eager run, graph re-capture) before its timed calls, which then all replay the graph.  Prints one JSON line: captions/s per arm and round, the median
ratio, the engine launches per batch of each arm, and the device name and power limit the numbers were measured at.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)


def device_info():
    info = {'device': torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        info['power_limit_and_max_sm_clock'] = out[0] if out else None
    except Exception:
        info['power_limit_and_max_sm_clock'] = None
    return info


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--batch', type=int, default=256)
    p.add_argument('--beam', type=int, default=9)
    p.add_argument('--groups', type=int, default=3)
    p.add_argument('--steps', type=int, default=10)
    p.add_argument('--warmup', type=int, default=3)
    p.add_argument('--rounds', type=int, default=3)
    p.add_argument('--mode', default='tc_f16x3', choices=['tc_f16x3', 'tc_f16x1', 'simt_fp32'])
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('dbs_rate.py measures on a CUDA device; none is visible')
    from imagecaptioning.pytorch_b200 import synthetic as syn
    cfg = dict(V=9487, E=1000, H=1000, A=512, F_fc=2048, F_att=2048, T=20)
    model = syn.build_model('updown', seed=1234, logit_scale=12.0, mode=a.mode, device=torch.device('cuda:0'), **cfg)
    fc, att = syn.make_inputs(a.batch, 36, cfg['F_fc'], cfg['F_att'], seed=1234)
    fc, att = fc.cuda(), att.cuda()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    arms = {'plain': {'beam_size': a.beam, 'sample_n': 1},
            'diverse': {'beam_size': a.beam, 'group_size': a.groups, 'diversity_lambda': 0.5, 'sample_n': 1}}
    rates = {k: [] for k in arms}
    launches = {}
    with torch.no_grad(), torch.cuda.stream(side):
        for name, opt in arms.items():              # warm-up: eager run, graph capture, replays
            for _ in range(a.warmup):
                model(fc, att, None, opt=opt, mode='sample')
            torch.cuda.synchronize()
            l0 = model.launch_count
            model(fc, att, None, opt=opt, mode='sample')
            torch.cuda.synchronize()
            launches[name] = model.launch_count - l0
        for _ in range(a.rounds):
            for name, opt in arms.items():
                # the engine keeps one captured loop: after the other arm ran, the first call is eager and the second re-captures
                for _ in range(2):
                    model(fc, att, None, opt=opt, mode='sample')
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(a.steps):
                    model(fc, att, None, opt=opt, mode='sample')
                torch.cuda.synchronize()
                rates[name].append(a.batch * a.steps / (time.perf_counter() - t0))
    ratio = statistics.median(d / p_ for d, p_ in zip(rates['diverse'], rates['plain']))
    print(json.dumps({'metric': 'captions_per_s', 'model': 'updown', 'dims': 'configs[1]', 'batch': a.batch, 'beam': a.beam, 'groups': a.groups,
                      'mode': a.mode, 'steps': a.steps, 'plain': [round(x, 1) for x in rates['plain']],
                      'diverse': [round(x, 1) for x in rates['diverse']], 'diverse_over_plain': round(ratio, 3),
                      'launches_per_batch': launches, **device_info()}))


if __name__ == '__main__':
    main()
