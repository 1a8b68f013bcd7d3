"""Generate tests/golden/corpus_cider.npz from the LIVE reference (build container only; the reference checkout is read-only).

    python tests/make_corpus_golden.py        # needs the reference checkout that oracle/make_golden.py reads

The reference's captioning/utils/rewards.py runs unmodified after init_scorer('corpus'), i.e. CiderD(df='corpus'): the document
frequencies come from the references of each call (ciderD_scorer.py:143-147, 182-186, 210-216).  At configs[3] size (10 images x 5 samples
+ greedy, 5 references each, V = 9487, T = 16) the file holds, for every weight pair in `weights`:
  reward_<j>  get_self_critical_reward (each image counted n + 1 times: n samples and its greedy caption)
  scores_<j>  get_scores (each image counted n times)
plus the inputs gts [B, 5, T], sampled [B*n, T], greedy [B, T].
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
sys.path.insert(0, REPO)
sys.path.insert(0, HERE)

from oracle import ciderd_oracle as cdo                         # noqa: E402
from oracle.make_golden import _enter_scratch                    # noqa: E402

WEIGHTS = [(1.0, 0.0), (0.7, 0.3), (2.0, 0.5)]
V, B, N_PER, T = 9487, 10, 5, 16


def main():
    out = os.path.join(HERE, 'golden', 'corpus_cider.npz')
    _enter_scratch()
    from captioning.utils import rewards as R
    R.CiderD_scorer = None
    R.Cider_scorer = None
    R.init_scorer('corpus')
    gts = cdo.make_refs(B, V, seed=23, L=T)
    rng = np.random.RandomState(9)

    def rows(k):
        o = np.zeros((k, T), np.int64)
        for i in range(k):
            ln = rng.randint(1, T + 1)
            o[i, :ln] = np.minimum(rng.zipf(1.3, size=ln), V)
        return o
    sampled, greedy = rows(B * N_PER), rows(B)
    for i in range(B):                                              # pieces of the references: non-trivial scores
        sampled[i * N_PER, :7] = gts[i][0][:7]
        sampled[i * N_PER + 1, :10] = gts[i][2][:10]
        sampled[i * N_PER + 2, :4] = gts[(i + 1) % B][1][:4]        # another image's n-gram: counted in df, not in this image's refs
        greedy[i, :5] = gts[i][1][:5]
    res = {'gts': np.stack(gts), 'sampled': sampled, 'greedy': greedy, 'weights': np.array(WEIGHTS), 'meta': np.array([V, B, N_PER, T])}
    for j, (wc, wb) in enumerate(WEIGHTS):
        opt = argparse.Namespace(cider_reward_weight=wc, bleu_reward_weight=wb)
        res['reward_%d' % j] = np.asarray(R.get_self_critical_reward(torch.from_numpy(greedy), gts, torch.from_numpy(sampled), opt), np.float64)
        res['scores_%d' % j] = np.asarray(R.get_scores(gts, torch.from_numpy(sampled), opt), np.float64) * np.ones(B * N_PER)
    np.savez_compressed(out, **res)
    print('corpus_cider: %d weight pairs, mean |reward| %.4f' % (len(WEIGHTS), float(np.abs(res['reward_0']).mean())))


if __name__ == '__main__':
    main()
