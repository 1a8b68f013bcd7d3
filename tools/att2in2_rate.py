"""Throughput of the Att2in2 family at the a2i2 recipe dimensions (E = H = A = 512, V = 9487, T = 20, 36 regions of 2048 features).

    python tools/att2in2_rate.py [--batch 256] [--beam 5] [--steps 10] [--warmup 3] [--scst-steps 20] [--mode tc_f16x3]

Two measurements on synthetic, seeded, device-resident inputs, each timed window ending in a device synchronise:
* decode: beam search at batch 256, beam 5, on a side stream where the engine captures the beam loop into a CUDA graph and replays it;
* train: the fused SCST step at 10 images x 5 samples (the a2i2_sc recipe's batch_size / train_sample_n), greedy baseline, dropout 0.5,
  replayed from its step graph after the eager and capturing calls.
Prints one JSON line with both rates, the engine launches per call and the device name and power limit they were measured at.
"""
from __future__ import annotations

import json
import os
import sys
import time
import argparse

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tools'))

from dbs_rate import device_info      # noqa: E402


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--batch', type=int, default=256)
    p.add_argument('--beam', type=int, default=5)
    p.add_argument('--steps', type=int, default=10)
    p.add_argument('--warmup', type=int, default=3)
    p.add_argument('--scst-steps', type=int, default=20)
    p.add_argument('--mode', default='tc_f16x3', choices=['tc_f16x3', 'tc_f16x1', 'simt_fp32'])
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('att2in2_rate.py measures on a CUDA device; none is visible')
    from imagecaptioning.pytorch_b200 import synthetic as syn
    from imagecaptioning.pytorch_b200 import rewards
    cfg = dict(V=9487, E=512, H=512, A=512, F_fc=2048, F_att=2048, T=20)
    model = syn.build_model('att2in2', seed=1234, logit_scale=12.0, mode=a.mode, device=torch.device('cuda:0'), **cfg)
    fc, att = syn.make_inputs(a.batch, 36, cfg['F_fc'], cfg['F_att'], seed=1234)
    fc, att = fc.cuda(), att.cuda()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    opt = {'beam_size': a.beam, 'sample_n': 1}
    with torch.no_grad(), torch.cuda.stream(side):
        for _ in range(a.warmup):
            model(fc, att, None, opt=opt, mode='sample')
        torch.cuda.synchronize()
        l0 = model.launch_count
        t0 = time.perf_counter()
        for _ in range(a.steps):
            model(fc, att, None, opt=opt, mode='sample')
        torch.cuda.synchronize()
        decode_rate = a.batch * a.steps / (time.perf_counter() - t0)
        decode_launches = (model.launch_count - l0) / a.steps
    # SCST step, 10 images x 5 samples
    B, n = 10, 5
    refs = syn.make_refs(200, cfg['V'], seed=4)
    df, ref_len = syn.document_frequency(refs)
    table = rewards.CiderDTable(df, ref_len)
    gts = refs[:B]
    sfc, satt = fc[:B].contiguous(), att[:B].contiguous()
    model.train()
    for i in range(3):                     # eager, capture, first replay
        model.scst_step(sfc, satt, gts, table, n, seed=i)
    torch.cuda.synchronize()
    l0 = model.launch_count
    t0 = time.perf_counter()
    for i in range(a.scst_steps):
        model.scst_step(sfc, satt, gts, table, n, seed=100 + i)
    torch.cuda.synchronize()
    dt = (time.perf_counter() - t0) / a.scst_steps
    print(json.dumps({'model': 'att2in2', 'dims': 'a2i2 recipe (E=H=A=512, V=9487, T=20, R=36)', 'mode': a.mode,
                      'decode': {'batch': a.batch, 'beam': a.beam, 'captions_per_s': round(decode_rate, 1), 'launches_per_batch': decode_launches},
                      'scst': {'images': B, 'sample_n': n, 'ms_per_step': round(1e3 * dt, 3), 'samples_per_s': round(B * n / dt, 1),
                               'launches_per_step': (model.launch_count - l0) / a.scst_steps},
                      **device_info()}))


if __name__ == '__main__':
    main()
