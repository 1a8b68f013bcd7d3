"""Cost of the BLEU-4 reward term and of the reward weights.

    python tools/reward_rate.py [--steps 20] [--windows 5]

* reward: the standalone device reward (rewards.weighted_scores with the greedy baseline, weights (0.5, 0.5): CIDEr-D + BLEU-4 + combine +
  reward) at 60 hypotheses x 5 references (10 images x 5 samples + greedy) and at 4000 x 50 (the hypothesis count of a large eval
  batch, 50 references each: the PASCAL-50S reference count), ms per call as the median over --windows windows of --steps calls.  Beside
  it, the reference's CPU get_self_critical_reward with the same weights, from oracle/_ref/ when that copy is present (60 x 5 only).
* steps: the AoANet SCST step at BASELINE configs[3] (configs/aoa.yml: E = H = 1024, 8 heads) and the UpDown SCST step (bench.py's
  dimensions), 10 images x 5 samples, with weights (1, 0) and (0.5, 0.5) alternated window by window in the same run; ms per step as
  the median over the windows of each weight pair (>= 20 steps per window), and launches per step.
Prints one JSON line with the device name and power limit of the same run.
"""
from __future__ import annotations

import argparse
import collections
import contextlib
import io
import json
import os
import pickle
import shutil
import statistics
import sys
import tempfile
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tools'))

import bench                          # noqa: E402
from dbs_rate import device_info      # noqa: E402


def windows(fn, steps, n_windows, sync=True):
    ms = []
    for w in range(n_windows):
        t0 = time.perf_counter()
        for i in range(steps):
            fn(w * steps + i)
        if sync:
            torch.cuda.synchronize()
        ms.append(1e3 * (time.perf_counter() - t0) / steps)
    return ms


def summary(ms):
    return {'ms': round(statistics.median(ms), 4), 'ms_min': round(min(ms), 4), 'ms_max': round(max(ms), 4)}


def hyps(rng, k, T, V):
    out = np.zeros((k, T), np.int64)
    for i in range(k):
        ln = rng.randint(4, T)
        out[i, :ln] = np.minimum(rng.zipf(1.3, size=ln), V)
    return out


def reward_rate(a, syn, rewards, table, V):
    res = {}
    rng = np.random.RandomState(3)
    for B, n, nref in ((10, 5, 5), (666, 5, 50)):          # 60 and 3996 hypotheses
        T = 16
        gts = syn.make_refs(B, V, n_refs=nref, seed=5)
        sampled = torch.from_numpy(hyps(rng, B * n, T, V)).cuda()
        greedy = torch.from_numpy(hyps(rng, B, T, V)).cuda()
        call = lambda _: rewards.weighted_scores(gts, sampled, (0.5, 0.5), greedy_res=greedy, with_reward=True)      # noqa: E731
        for i in range(3):
            call(i)
        torch.cuda.synchronize()
        key = '%dx%d' % (B * n + B, nref)
        res[key] = summary(windows(call, a.steps, a.windows))
        res[key]['hypotheses'] = B * n + B
    # the reference's host path at the small shape: the unmodified modules of the oracle/_ref copy, imported from a scratch directory that
    # holds the cwd-relative names they expect (cider, coco-caption, data/<df>.p; captioning/utils/rewards.py:12,15)
    ref = os.path.join(REPO, 'oracle', '_ref')
    if not os.path.isdir(os.path.join(ref, 'captioning')):
        res['reference_cpu_60x5'] = 'oracle/_ref/ not present'
        return res
    scratch = tempfile.mkdtemp(prefix='refcwd_')
    try:
        for name in ('cider', 'coco-caption'):
            os.symlink(os.path.join(ref, name), os.path.join(scratch, name))
        os.makedirs(os.path.join(scratch, 'data'))
        df, ref_len = syn.document_frequency(syn.make_refs(200, V, seed=4))
        dd = collections.defaultdict(float)
        dd.update({tuple(str(t) for t in k): float(v) for k, v in df.items()})
        with open(os.path.join(scratch, 'data', 'rate-df.p'), 'wb') as f:
            pickle.dump({'document_frequency': dd, 'ref_len': ref_len}, f, protocol=2)
        os.chdir(scratch)
        sys.path.insert(0, ref)
        with contextlib.redirect_stdout(io.StringIO()):                   # the reference prints every score
            from captioning.utils import rewards as R
            R.init_scorer('rate-df')
            gts = syn.make_refs(10, V, n_refs=5, seed=5)
            s, g = torch.from_numpy(hyps(rng, 50, 16, V)), torch.from_numpy(hyps(rng, 10, 16, V))
            opt = argparse.Namespace(cider_reward_weight=0.5, bleu_reward_weight=0.5)
            res['reference_cpu_60x5'] = summary(windows(lambda _: R.get_self_critical_reward(g, gts, s, opt), 5, 3, sync=False))
    except Exception as e:              # the reference copy is optional: report, do not fail the device numbers
        res['reference_cpu_60x5'] = 'failed: %r' % e
    finally:
        os.chdir(REPO)
        shutil.rmtree(scratch, ignore_errors=True)
    return res


def step_rate(a, syn, rewards, table, refs):
    res = {}
    B, n = 10, 5
    fc, att = syn.make_inputs(B, 36, 2048, 2048, seed=1)
    fc, att = fc.cuda(), att.cuda()
    gts = refs[:B]
    for fam in ('aoa', 'updown'):
        if fam == 'aoa':
            model = syn.build_model('aoa', seed=1234, logit_scale=6.0, mode='tc_f16x3', device='cuda', heads=8, **dict(bench.CFG, E=1024, H=1024, A=0))
        else:
            model = syn.build_model('updown', seed=1234, logit_scale=12.0, mode='tc_f16x3', device='cuda', **bench.CFG)
        model.train()
        per = {'1,0': [], '0.5,0.5': []}
        launches = {}
        weights = {'1,0': None, '0.5,0.5': (0.5, 0.5)}
        for key, w in weights.items():             # eager, capture and first replay of each configuration
            for s in range(3):
                model.scst_step(fc, att, gts, table, n, seed=s, reward_weights=w)
        torch.cuda.synchronize()
        for win in range(2 * a.windows):
            key = '1,0' if win % 2 == 0 else '0.5,0.5'
            l0 = model.launch_count
            per[key] += windows(lambda s: model.scst_step(fc, att, gts, table, n, seed=100 + s, reward_weights=weights[key]), a.steps, 1)
            launches[key] = (model.launch_count - l0) / a.steps
        res[fam] = {k: dict(summary(v), launches_per_step=launches[k]) for k, v in per.items()}
        del model
        torch.cuda.empty_cache()
    return res


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--steps', type=int, default=20)
    p.add_argument('--windows', type=int, default=5)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('reward_rate.py measures on a CUDA device; none is visible')
    a.steps = max(a.steps, 20)
    from imagecaptioning.pytorch_b200 import rewards
    from imagecaptioning.pytorch_b200 import synthetic as syn
    V = bench.CFG['V']
    refs = syn.make_refs(200, V, seed=4)
    table = rewards.CiderDTable(*syn.document_frequency(refs))
    rewards.reset_scorer()
    rewards.init_scorer(table)
    out = {'reward': reward_rate(a, syn, rewards, table, V), 'scst_step': step_rate(a, syn, rewards, table, refs), 'steps_per_window': a.steps,
           'windows': a.windows}
    out.update(device_info())
    print(json.dumps(out))


if __name__ == '__main__':
    main()
