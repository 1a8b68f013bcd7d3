"""Cost of region counts past the staged attention kernels' shared-memory limit.

1. The attention operations alone (capb200_mha_forward in its training form with dropout 0.1, capb200_mha_self_backward and
   capb200_mha_cross_backward with 5 rows per image), 10 images x 8 heads at head widths 64 and 128, staged (form 1, where it fits) and
   key-tiled (form 2), so the cost of the switch shows on both sides of it.  CUDA events around `--launches` launches.
2. The AoANet self-critical step of BASELINE configs[3] (10 images x 5 samples, E = H = 1024, 8 heads, T = 20, tc_f16x3) at R in
   {36, 75, 76, 100, 196}: 75 is the last count the staged refiner backward holds at head width 128.
3. The Transformer 6 + 6 / d_model 512 / 8 heads XE step (10 images x 5 captions) and self-critical step (10 x 5) at R in {36, 105, 106, 196}.
Steps are timed with a host clock around `--steps` calls ending in a device synchronise.

Prints one JSON line with the card name and power limit read in the same run.

    python tools/region_rate.py [--launches 50] [--repeats 5] [--steps 5] [--skip-model]
"""
import argparse
import json
import os
import statistics
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tools'))

from dbs_rate import device_info            # noqa: E402
from large_vocab_rate import timed          # noqa: E402

HEADS, B = 8, 10
LIMIT = 200 * 1024
CFG = dict(V=9487, F_fc=2048, F_att=2048, T=20)


def staged_fits(op, R, dk, rows=0):
    f = {'forward': 2 * R * (dk + 4) + 8 * R + 8 * dk, 'self_backward': 4 * R * (dk + 4) + 2 * R * R,
         'cross_backward': 2 * R * (dk + 1) + 2 * rows * (dk + 1) + 2 * rows * R}[op]
    return 4 * f <= LIMIT


def op_ms(L, op, form, R, dk, launches, repeats):
    lib, st = L.load(), L.current_stream()
    H = HEADS * dk
    g = torch.Generator(device='cuda').manual_seed(R + dk)
    x = [torch.randn(B * R, H, device='cuda', generator=g) for _ in range(7)]
    rpi = 5
    qx, dox, dqx = (torch.randn(B * rpi, H, device='cuda', generator=g) for _ in range(3))
    probs = torch.softmax(torch.randn(B * rpi * HEADS, R, device='cuda', generator=g), -1)

    def launch():
        if op == 'forward':
            rc = lib.capb200_mha_forward(form, 1, B, R, HEADS, dk, L.ptr(x[0]), L.ptr(x[1]), L.ptr(x[2]), H, None, 0, 7, 11, 0.1, L.ptr(x[3]), H, st)
        elif op == 'self_backward':
            rc = lib.capb200_mha_self_backward(form, B, R, HEADS, dk, L.ptr(x[0]), L.ptr(x[1]), L.ptr(x[2]), H, None, 0, 7, 11, 0.1, L.ptr(x[3]), H,
                                               L.ptr(x[4]), L.ptr(x[5]), L.ptr(x[6]), H, st)
        else:
            rc = lib.capb200_mha_cross_backward(form, B, rpi, 1, HEADS, dk, R, L.ptr(qx), H, L.ptr(x[1]), L.ptr(x[2]), H, 7, 5, 0, 0.1, L.ptr(probs),
                                                L.ptr(dox), H, L.ptr(dqx), H, L.ptr(x[5]), L.ptr(x[6]), H, st)
        L.check(rc, op)

    for _ in range(5):
        launch()
    torch.cuda.synchronize()
    ms = []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(launches):
            launch()
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1) / launches)
    return {'ms': round(statistics.median(ms), 4), 'min': round(min(ms), 4), 'max': round(max(ms), 4)}


def op_table(L, launches, repeats):
    out = {}
    for dk in (64, 128):
        for R in (36, 75, 76, 105, 106, 196, 577):
            for op in ('forward', 'self_backward', 'cross_backward'):
                forms = ((1, 'staged'), (2, 'tiled')) if staged_fits(op, R, dk, 5) else ((2, 'tiled'),)
                for form, name in forms:
                    out['%s dk=%d R=%d %s' % (op, dk, R, name)] = op_ms(L, op, form, R, dk, launches, repeats)
    return out


def model_table(steps, repeats):
    import imagecaptioning.pytorch_b200 as b200
    from imagecaptioning.pytorch_b200 import synthetic as syn
    dev = torch.device('cuda:0')
    refs = syn.make_refs(200, CFG['V'], seed=4)
    table = b200.rewards.CiderDTable(*syn.document_frequency(refs))
    out = {}
    model = syn.build_model('aoa', seed=1234, logit_scale=6.0, mode='tc_f16x3', device=dev, heads=8, **dict(CFG, E=1024, H=1024, A=0))
    model.train()
    for R in (36, 75, 76, 100, 196):
        fc, att = (t.cuda() for t in syn.make_inputs(B, R, CFG['F_fc'], CFG['F_att'], seed=R))
        out['aoa scst_step 10x5 R=%d' % R] = timed(lambda: model.scst_step(fc, att, refs[:B], table, 5), steps, 2, repeats)
    del model
    torch.cuda.empty_cache()
    model = syn.build_model('transformer', seed=1234, logit_scale=3.0, mode='tc_f16x3', device=dev, heads=8, **dict(CFG, E=512, H=2048, A=6))
    model.train()
    g = torch.Generator().manual_seed(5)
    T = CFG['T']
    labels = torch.zeros(B, 5, T + 2, dtype=torch.long)
    labels[..., 1:T + 1] = torch.randint(1, CFG['V'] + 1, (B, 5, T), generator=g)
    masks = torch.ones(B, 5, T + 2)
    labels, masks = labels.cuda(), masks.cuda()
    for R in (36, 105, 106, 196):
        fc, att = (t.cuda() for t in syn.make_inputs(B, R, CFG['F_fc'], CFG['F_att'], seed=R))
        out['transformer xe_step 10x5 R=%d' % R] = timed(lambda: model.xe_step(fc, att, labels, masks), steps, 2, repeats)
        out['transformer scst_step 10x5 R=%d' % R] = timed(lambda: model.scst_step(fc, att, refs[:B], table, 5), steps, 2, repeats)
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--launches', type=int, default=50)
    p.add_argument('--repeats', type=int, default=5)
    p.add_argument('--steps', type=int, default=5)
    p.add_argument('--skip-model', action='store_true')
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('region_rate.py measures on a CUDA device; none is visible')
    import imagecaptioning.pytorch_b200 as b200
    out = {'images': B, 'heads': HEADS, 'launches_per_window': a.launches, 'windows': a.repeats}
    out['attention_ms_per_launch'] = op_table(b200._lib, a.launches, a.repeats)
    if not a.skip_model:
        out['steps'] = model_table(a.steps, a.repeats)
    out.update(device_info())
    print(json.dumps(out))


if __name__ == '__main__':
    main()
