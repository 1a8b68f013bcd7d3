"""Cost of AttModel's multi-layer output head (logit_layers = k) on the engine, at k = 1, 2 and 3:
* UpDown beam-5 decode at batch 256 with BASELINE configs[1]'s dimensions (V = 9487, E = H = 1000, A = 512, 2048-d features, 36 regions,
  T = 20).  Each hidden layer adds one [rows, H] x [H, H] GEMM per step, about H / (V + 1) = 10.5 % of the vocabulary GEMM's FLOPs here;
* UpDown's fused self-critical step at recipe size (10 images x 5 samples, V = 9487, E = H = A = 512, T = 16, 36 regions), which runs the head
  in the greedy baseline, in the train-mode sampled pass with its dropout, and in the batched backward.
Prints one JSON line with the card name and power limit read in the same run.

    python tools/logit_layers_rate.py [--steps 5] [--warmup 2] [--repeats 5] [--batch 256]
"""
import argparse
import json
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tools'))

from autograd_rate import timed       # noqa: E402
from dbs_rate import device_info      # noqa: E402

CFG = dict(V=9487, E=1000, H=1000, A=512, F_fc=2048, F_att=2048, T=20)
RECIPE = dict(V=9487, E=512, H=512, A=512, F_fc=2048, F_att=2048, T=16)
R = 36


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--steps', type=int, default=5)
    p.add_argument('--warmup', type=int, default=2)
    p.add_argument('--repeats', type=int, default=5)
    p.add_argument('--batch', type=int, default=256)
    p.add_argument('--mode', default='tc_f16x3', choices=['tc_f16x3', 'tc_f16x1', 'simt_fp32'])
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('logit_layers_rate.py measures on a CUDA device; none is visible')
    from imagecaptioning.pytorch_b200 import synthetic as syn
    fc, att = syn.make_inputs(a.batch, R, CFG['F_fc'], CFG['F_att'], seed=1234)
    fc, att = fc.cuda(), att.cuda()
    out = {'workload': 'updown beam 5', 'images': a.batch, 'regions': R, 'dims': CFG, 'mode': a.mode, 'steps_per_window': a.steps,
           'windows': a.repeats, 'beam5': {}}
    for k in (1, 2, 3):
        model = syn.build_model('updown', seed=1234, logit_scale=12.0, mode=a.mode, device=torch.device('cuda:0'), logit_layers=k, **CFG)

        def decode():
            with torch.no_grad():
                model(fc, att, None, opt={'beam_size': 5, 'sample_n': 1}, mode='sample')
        res = timed(decode, a.steps, max(3, a.warmup), a.repeats)       # >= 3 warm-up calls: eager, graph capture, first replay
        res['captions_per_s'] = round(a.batch / (res['ms_per_step'] / 1e3), 1)
        out['beam5']['k%d' % k] = res
        del model
        torch.cuda.empty_cache()
    base = out['beam5']['k1']['ms_per_step']
    for k in (2, 3):
        out['beam5']['k%d_over_k1' % k] = round(out['beam5']['k%d' % k]['ms_per_step'] / base, 3)
    from imagecaptioning.pytorch_b200 import rewards
    Bs, n = 10, 5
    fc, att = syn.make_inputs(Bs, R, RECIPE['F_fc'], RECIPE['F_att'], seed=1234)
    fc, att = fc.cuda(), att.cuda()
    refs = syn.make_refs(200, RECIPE['V'], seed=4)
    table = rewards.CiderDTable(*syn.document_frequency(refs))
    out['scst_step'] = {'workload': 'updown scst step (greedy baseline)', 'images': Bs, 'per_image': n, 'dims': RECIPE}
    for k in (1, 2, 3):
        model = syn.build_model('updown', seed=1234, logit_scale=12.0, mode=a.mode, device=torch.device('cuda:0'), logit_layers=k, **RECIPE)
        model.train()
        # >= 3 warm-up calls of the step: eager, graph capture, first replay
        out['scst_step']['k%d' % k] = timed(lambda: model.scst_step(fc, att, refs[:Bs], table, n), a.steps, max(3, a.warmup), a.repeats)
        del model
        torch.cuda.empty_cache()
    base = out['scst_step']['k1']['ms_per_step']
    for k in (2, 3):
        out['scst_step']['k%d_over_k1' % k] = round(out['scst_step']['k%d' % k]['ms_per_step'] / base, 3)
    out.update(device_info())
    print(json.dumps(out))


if __name__ == '__main__':
    main()
