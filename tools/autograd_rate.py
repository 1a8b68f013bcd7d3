"""Cost of the autograd path (model.autograd) against the fused training steps, at recipe size: one XE step and one new_self_critical step
of UpDown (configs/updown: E = H = A = 512, F = 2048) and of the Transformer (d_model 512, d_ff 2048, 6 + 6 layers, 8 heads), V = 9487,
10 images x 5 captions / samples, T = 16.  The autograd XE step is LanguageModelCriterion on model(fc, att, labels[..., :-1]) and
backward(); the autograd new_self_critical step is the train-mode sample, the engine's CIDEr-D scores and the leave-one-out criterion in
PyTorch, and backward().  Also the kernel time of logsoftmax_vjp (torch.profiler, a separate pass).  Prints one JSON line with the card
name and power limit read in the same run.

    python tools/autograd_rate.py [--steps 10] [--warmup 3] [--repeats 5] [--mode tc_f16x3]
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

DIMS = {'updown': dict(V=9487, E=512, H=512, A=512, F_fc=2048, F_att=2048, T=16),
        'transformer': dict(V=9487, E=512, H=2048, A=6, F_fc=2048, F_att=2048, T=16)}


def timed(step, steps, warmup, repeats):
    for i in range(warmup):
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


def lm_criterion(lp, target, mask):
    L = lp.shape[1]
    target, mask = target.reshape(-1, target.shape[-1])[:, :L], mask.reshape(-1, mask.shape[-1])[:, :L]
    return -(lp.gather(2, target.unsqueeze(2)).squeeze(2) * mask).sum() / mask.sum()


def nsc_criterion(lp, seq, scores, n):
    mask = torch.cat([torch.ones_like(seq[:, :1]), (seq[:, :-1] > 0).long()], 1).to(lp)
    sc = scores.to(lp).view(-1, n)
    sc = (sc - (sc.sum(1, keepdim=True) - sc) / (n - 1)).reshape(-1, 1)
    return -(lp.gather(2, seq.unsqueeze(2)).squeeze(2) * mask * sc).sum() / mask.sum()


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--steps', type=int, default=10)
    p.add_argument('--warmup', type=int, default=3)
    p.add_argument('--repeats', type=int, default=5)
    p.add_argument('--mode', default='tc_f16x3', choices=['tc_f16x3', 'simt_fp32'])
    p.add_argument('--families', default='updown,transformer')
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('autograd_rate.py measures on a CUDA device; none is visible')
    from imagecaptioning.pytorch_b200 import rewards
    from imagecaptioning.pytorch_b200 import synthetic as syn
    B, n, R = 10, 5, 36
    out = {'images': B, 'per_image': n, 'regions': R, 'mode': a.mode, 'steps_per_window': a.steps, 'windows': a.repeats}
    for family in a.families.split(','):
        cfg = DIMS[family]
        model = syn.build_model(family, seed=1234, logit_scale=12.0, mode=a.mode, device=torch.device('cuda:0'), heads=8, **cfg)
        model.autograd = True
        model.train()
        fc, att = syn.make_inputs(B, R, cfg['F_fc'], cfg['F_att'], seed=1234)
        fc, att = fc.cuda(), att.cuda()
        refs = syn.make_refs(200, cfg['V'], seed=4)
        table = rewards.CiderDTable(*syn.document_frequency(refs))
        gts = refs[:B]
        L = cfg['T'] + 2
        g = torch.Generator().manual_seed(12)
        labels = torch.zeros(B, n, L, dtype=torch.long)
        masks = torch.zeros(B, n, L)
        for i in range(B):
            for j in range(n):
                k = int(torch.randint(6, L - 1, (1,), generator=g))
                labels[i, j, 1:1 + k] = torch.randint(1, cfg['V'] + 1, (k,), generator=g)
                masks[i, j, :k + 2] = 1
        labels, masks = labels.cuda(), masks.cuda()

        def xe_autograd():
            model.zero_grad(set_to_none=True)
            lm_criterion(model(fc, att, labels[..., :-1]), labels[..., 1:], masks[..., 1:]).backward()

        def nsc_autograd():
            model.zero_grad(set_to_none=True)
            seq, lp = model(fc, att, None, opt={'sample_method': 'sample', 'sample_n': n, 'beam_size': 1}, mode='sample')
            nsc_criterion(lp, seq, rewards.cider_scores(gts, seq, table), n).backward()

        res = {'dims': cfg}
        res['xe_fused'] = timed(lambda: model.xe_step(fc, att, labels, masks), a.steps, a.warmup, a.repeats)
        res['xe_autograd'] = timed(xe_autograd, a.steps, a.warmup, a.repeats)
        # >= 3 warm-up calls of the fused step: eager, capture, first replay
        res['nsc_fused'] = timed(lambda: model.scst_step(fc, att, gts, table, n, baseline='leave_one_out'), a.steps, max(3, a.warmup), a.repeats)
        res['nsc_autograd'] = timed(nsc_autograd, a.steps, a.warmup, a.repeats)
        for k in ('xe', 'nsc'):
            res[k + '_autograd_over_fused'] = round(res[k + '_autograd']['ms_per_step'] / res[k + '_fused']['ms_per_step'], 3)
        # kernel time of logsoftmax_vjp: its launches in one autograd XE and one autograd new_self_critical step, profiled separately
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            xe_autograd()
            nsc_autograd()
            torch.cuda.synchronize()
        ks = [e for e in prof.events() if 'logsoftmax_vjp' in e.name and e.device_type.name == 'CUDA']
        res['logsoftmax_vjp'] = {'launches': len(ks), 'us_total': round(sum(e.device_time for e in ks), 1),
                                 'rows': [B * n * (L - 1), B * n * cfg['T']], 'V1': cfg['V'] + 1}
        out[family] = res
        del model
        torch.cuda.empty_cache()
    out.update(device_info())
    print(json.dumps(out))


if __name__ == '__main__':
    main()
