"""Cost of the fused PPO step (model.ppo_step: capb200_*_ppo_step) at recipe size, 10 images x 5 samples, T = 16, V = 9487, for every
family, against (a) the fused new_self_critical step (scst_step with the leave-one-out baseline, the same sampled forward without the old
policy) and (b) the autograd route: model.autograd = 1, the train-mode sample through autograd, the frozen old policy's teacher-forced
pass, the engine's CIDEr-D scores and the PPO criterion in PyTorch, and backward().  Prints one JSON line with the card name and power
limit read in the same run.

    python tools/ppo_rate.py [--steps 10] [--warmup 3] [--repeats 5] [--families updown,att2in2,newfc,aoa,transformer]
"""
import argparse
import copy
import json
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tools'))

from autograd_rate import timed       # noqa: E402
from dbs_rate import device_info      # noqa: E402

RNN = dict(V=9487, E=512, H=512, A=512, F_fc=2048, F_att=2048, T=16)
DIMS = {'updown': RNN, 'att2in2': RNN, 'newfc': RNN, 'aoa': dict(RNN, E=1024, H=1024),
        'transformer': dict(V=9487, E=512, H=2048, A=6, F_fc=2048, F_att=2048, T=16)}


def ppo_criterion(lp, lo, seq, scores, n, eps=0.2, kl_coef=0.02):
    """PPOLoss (losses.py:291-357), reduction 'mean', as host-level torch ops."""
    mask = torch.cat([torch.ones_like(seq[:, :1]), (seq[:, :-1] > 0).long()], 1).to(lp)
    sc = scores.to(lp).view(-1, n)
    adv = (sc - (sc.sum(1, keepdim=True) - sc) / (n - 1)).reshape(-1, 1)
    ratio = torch.exp((lp - lo).gather(2, seq.unsqueeze(2)).squeeze(2))
    pg = torch.max(-adv * ratio, -adv * ratio.clamp(1 - eps, 1 + eps))
    kl = (lo.exp() * (lo - lp)).sum(2)
    return ((pg + kl_coef * kl) * mask).sum() / mask.sum()


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--steps', type=int, default=10)
    p.add_argument('--warmup', type=int, default=3)
    p.add_argument('--repeats', type=int, default=5)
    p.add_argument('--mode', default='tc_f16x3', choices=['tc_f16x3', 'simt_fp32'])
    p.add_argument('--families', default='updown,att2in2,newfc,aoa,transformer')
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('ppo_rate.py measures on a CUDA device; none is visible')
    from imagecaptioning.pytorch_b200 import rewards
    from imagecaptioning.pytorch_b200 import synthetic as syn
    B, n, R = 10, 5, 36
    out = {'images': B, 'per_image': n, 'regions': R, 'mode': a.mode, 'steps_per_window': a.steps, 'windows': a.repeats}
    for family in a.families.split(','):
        cfg = DIMS[family]
        model = syn.build_model(family, seed=1234, logit_scale=12.0, mode=a.mode, device=torch.device('cuda:0'), heads=8, **cfg)
        model.train()
        old = copy.deepcopy(model).eval()
        with torch.no_grad():
            for q in old.parameters():
                q.add_(0.01 * torch.randn_like(q))
                q.requires_grad_(False)
        fc, att = syn.make_inputs(B, R, cfg['F_fc'], cfg['F_att'], seed=1234)
        fc, att = fc.cuda(), att.cuda()
        if family == 'newfc':
            att = fc.new_zeros(B, 0, 0)
        refs = syn.make_refs(200, cfg['V'], seed=4)
        table = rewards.CiderDTable(*syn.document_frequency(refs))
        gts = refs[:B]

        def ppo_autograd():
            model.zero_grad(set_to_none=True)
            seq, lp = model(fc, att, None, opt={'sample_method': 'sample', 'sample_n': n, 'beam_size': 1}, mode='sample')
            with torch.no_grad():
                lo = old(fc, att, torch.cat([seq.new_zeros(seq.shape[0], 1), seq[:, :-1]], 1).view(B, n, -1), None)
            ppo_criterion(lp, lo, seq, rewards.cider_scores(gts, seq, table), n).backward()

        res = {'dims': cfg}
        res['ppo_fused'] = timed(lambda: model.ppo_step(old, fc, att, gts, table, n), a.steps, a.warmup, a.repeats)
        # >= 3 warm-up calls of the new_self_critical step: eager, capture, first replay
        res['nsc_fused'] = timed(lambda: model.scst_step(fc, att, gts, table, n, baseline='leave_one_out'), a.steps, max(3, a.warmup), a.repeats)
        model.autograd = True
        res['ppo_autograd'] = timed(ppo_autograd, a.steps, a.warmup, a.repeats)
        model.autograd = False
        res['ppo_fused_over_nsc_fused'] = round(res['ppo_fused']['ms_per_step'] / res['nsc_fused']['ms_per_step'], 3)
        res['ppo_autograd_over_ppo_fused'] = round(res['ppo_autograd']['ms_per_step'] / res['ppo_fused']['ms_per_step'], 3)
        out[family] = res
        del model, old
        torch.cuda.empty_cache()
    out.update(device_info())
    print(json.dumps(out))


if __name__ == '__main__':
    main()
