"""Generate tests/golden/long_captions.npz from the LIVE reference (build container only; the reference checkout is read-only).

    python tests/make_long_captions_golden.py        # needs the reference checkout that oracle/make_golden.py reads

CIDEr-D and BLEU-4 rewards of captions and references past 64 tokens, from the reference's own scorers run unmodified: coco-caption's
Bleu(4) and captioning/utils/rewards.py's get_self_critical_reward / get_scores, with a document-frequency pickle written here (the
scripts/prepro_ngrams.py format) and with init_scorer('corpus').  Over a 6-word vocabulary, so n-grams repeat inside and across rows:
  4 images x 3 samples + a greedy caption each, T = L = 256.  Hypotheses of 65, 100 and 256 tokens (the last without a closing 0) and a few
  short ones; pieces of the references copied in.  Image 0's references are 65, 100 and 256 tokens long, image 1 mixes 8 / 12 / 70 / 150 /
  255, image 2 holds 64 / 65 / 100 / 200 / 30 and image 3 five references of 100.
The file holds the inputs, the pickle's document frequencies (df_keys / df_vals / ref_len), per-hypothesis BLEU-4 (`bleu`, S + B rows:
samples, then greedy captions) and, for every weight pair of `weights`, reward_<j> / scores_<j> (pickle table) and creward_<j> / cscores_<j>
(corpus table).
"""
from __future__ import annotations

import argparse
import os
import pickle
import sys
from collections import defaultdict

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
sys.path.insert(0, REPO)
sys.path.insert(0, HERE)

from oracle import ciderd_oracle as cdo                         # noqa: E402
from oracle.make_golden import _enter_scratch                    # noqa: E402

WEIGHTS = [(1.0, 0.0), (0.0, 1.0), (0.7, 0.3)]
V, B, N_PER, T, L = 6, 4, 3, 256, 256
REF_LENS = [[65, 100, 256], [8, 12, 70, 150, 255], [64, 65, 100, 200, 30], [100] * 5]
HYP_LENS = [65, 100, 256, 65, 100, 256, 10, 200, 65, 100, 256, 1]
GREEDY_LENS = [100, 65, 256, 40]


def _row(rng, width, ln):
    r = np.zeros(width, np.int64)
    r[:ln] = rng.randint(1, V + 1, size=ln)
    return r


def make_case():
    rng = np.random.RandomState(256)
    gts = []
    for lens in REF_LENS:
        rows = np.stack([_row(rng, L, ln) for ln in lens])
        gts.append(rows)
    sampled = np.stack([_row(rng, T, ln) for ln in HYP_LENS])
    greedy = np.stack([_row(rng, T, ln) for ln in GREEDY_LENS])
    for i in range(B):                             # long pieces of the references: n-grams of every order match
        sampled[i * N_PER, 10:60] = gts[i][0][10:60]
        sampled[i * N_PER + 1, :40] = gts[i][-1][:40]
        greedy[i, 5:35] = gts[i][1][5:35]
    return gts, sampled, greedy


def _bleu(gts_rows, hyp_rows):
    sys.path.append('coco-caption')
    from pycocoevalcap.bleu.bleu import Bleu
    from captioning.utils.rewards import array_to_str
    gts = {i: [array_to_str(r) for r in rows] for i, rows in enumerate(gts_rows)}
    res = {i: [array_to_str(h)] for i, h in enumerate(hyp_rows)}
    _, scores = Bleu(4).compute_score(gts, res)
    return np.array(scores[3], np.float64)


def main():
    out = os.path.join(HERE, 'golden', 'long_captions.npz')
    scratch = _enter_scratch()
    from captioning.utils import rewards as R
    gts, sampled, greedy = make_case()
    extra = [np.stack([_row(np.random.RandomState(900 + i), L, 40 + 20 * (i % 10)) for _ in range(3)]) for i in range(40)]
    df, ref_len = cdo.build_document_frequency(gts + extra)
    dd = defaultdict(float)
    dd.update({tuple(str(t) for t in k): v for k, v in df.items()})
    with open(os.path.join(scratch, 'data', 'long-df.p'), 'wb') as f:
        pickle.dump({'document_frequency': dd, 'ref_len': ref_len}, f, protocol=2)
    hyps = np.concatenate([sampled, greedy], 0)
    res = {'gts': np.stack([np.pad(g, ((0, 5 - g.shape[0]), (0, 0))) for g in gts]), 'ref_counts': np.array([g.shape[0] for g in gts]),
           'sampled': sampled, 'greedy': greedy, 'weights': np.array(WEIGHTS), 'meta': np.array([V, B, N_PER, T, L]),
           'df_keys': np.array([list(k) + [-1] * (4 - len(k)) for k in df], np.int64), 'df_vals': np.array(list(df.values()), np.float64),
           'ref_len': np.array(float(ref_len)),
           'bleu': _bleu([gts[i // N_PER] for i in range(B * N_PER)] + list(gts), list(hyps))}
    for table in ('long-df', 'corpus'):
        R.CiderD_scorer = None
        R.Cider_scorer = None
        R.init_scorer(table)
        pre = '' if table == 'long-df' else 'c'
        for j, (wc, wb) in enumerate(WEIGHTS):
            opt = argparse.Namespace(cider_reward_weight=wc, bleu_reward_weight=wb)
            res['%sreward_%d' % (pre, j)] = np.asarray(R.get_self_critical_reward(torch.from_numpy(greedy), gts, torch.from_numpy(sampled), opt),
                                                       np.float64)
            res['%sscores_%d' % (pre, j)] = np.asarray(R.get_scores(gts, torch.from_numpy(sampled), opt), np.float64) * np.ones(B * N_PER)
    R.CiderD_scorer = None
    np.savez_compressed(out, **res)
    print('long_captions: %d hypotheses, mean BLEU-4 %.4f, CIDEr-D scores %s' % (len(hyps), res['bleu'].mean(), np.round(res['scores_0'], 4)))


if __name__ == '__main__':
    main()
