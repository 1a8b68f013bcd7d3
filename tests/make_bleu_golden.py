"""Generate tests/golden/bleu_reward.npz from the LIVE reference (build container only; the reference checkout is read-only).

    python tests/make_bleu_golden.py        # needs the reference checkout that oracle/make_golden.py reads

The reference's scorers are imported unmodified: coco-caption's Bleu(4) for the BLEU-4 term, and captioning/utils/rewards.py's
get_self_critical_reward / get_scores (CIDEr-D from a document-frequency pickle written here, in the scripts/prepro_ngrams.py format).
The file holds
  (a) syn_*   a few hundred synthetic hypothesis / reference-set pairs over a 6-word vocabulary: a hypothesis that is only "0", rows
              without a 0, n-grams repeated beyond the references' counts, ties of the closest reference length, hypotheses shorter and
              longer than every reference, images with 1 and with 5 to 40 references;  syn_bleu = Bleu(4).compute_score(...)[1][3];
  (b) pascal_bleu  BLEU-4 of the PASCAL-50S candidates of tests/golden/ciderd_pascal.npz against their 50 references (same id mapping);
  (c) full_*  get_self_critical_reward and get_scores at SCST shape (10 images x 5 samples + greedy, T = 20) for the weight pairs in
              full_weights, with the document frequencies the GPU test rebuilds the CIDEr-D table from.
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

WEIGHTS = [(0.7, 0.3), (0.0, 1.0), (2.0, 0.0), (1.0, 0.5), (-1.0, 1.0)]


def _bleu(gts_rows, hyp_rows):
    """Per-sentence BLEU-4 of the reference scorer: gts_rows[i] is a list of id rows, hyp_rows[i] one id row."""
    sys.path.append('coco-caption')
    from pycocoevalcap.bleu.bleu import Bleu
    from captioning.utils.rewards import array_to_str
    gts = {i: [array_to_str(r) for r in rows] for i, rows in enumerate(gts_rows)}
    res = {i: [array_to_str(h)] for i, h in enumerate(hyp_rows)}
    _, scores = Bleu(4).compute_score(gts, res)
    return np.array(scores[3], np.float64)


def _row(rng, T, ln, V, end=True):
    r = np.zeros(T, np.int64)
    r[:ln] = rng.randint(1, V + 1, size=ln)
    if not end:
        r[:] = rng.randint(1, V + 1, size=T)
    return r


def gen_synthetic(rng):
    V, T, L = 6, 16, 14
    hyps, ref_sets = [], []

    def add(h, refs):
        hyps.append(h)
        ref_sets.append(np.stack(refs))
    add(np.zeros(T, np.int64), [_row(rng, L, 5, V)])                                                 # hypothesis "0"
    add(np.zeros(T, np.int64), [np.zeros(L, np.int64), _row(rng, L, 3, V)])                          # "0" against a "0" reference
    add(_row(rng, T, 0, V, end=False), [_row(rng, L, 0, V, end=False)])                              # no 0 in either
    h = np.zeros(T, np.int64); h[:9] = 2                                                             # clipping: "2" x 9
    add(h, [np.array([2, 2, 3, 2, 0] + [0] * (L - 5)), np.array([2, 2, 2, 1, 0] + [0] * (L - 5))])
    h = np.zeros(T, np.int64); h[:4] = [1, 2, 3, 4]                                                  # testlen 5; references of length 4 and 6
    add(h, [np.array([1, 2, 3, 0] + [0] * (L - 4)), np.array([1, 2, 3, 4, 5, 0] + [0] * (L - 6))])
    add(h, [np.array([1, 2, 3, 4, 5, 0] + [0] * (L - 6)), np.array([4, 3, 0] + [0] * (L - 3)), np.array([1, 2, 3, 0] + [0] * (L - 4))])
    for _ in range(300):
        ln = rng.randint(0, T + 1)
        h = _row(rng, T, min(ln, T), V, end=ln < T)
        nref = [1, 1, 2, 5, 5, 7, 12, 40][rng.randint(0, 8)]
        kind = rng.randint(0, 4)
        refs = []
        for _ in range(nref):
            if kind == 0:                                           # references longer than the hypothesis (brevity penalty)
                rl = min(L, ln + 1 + rng.randint(0, 6))
            elif kind == 1:                                         # shorter
                rl = max(0, ln - 1 - rng.randint(0, 6))
            else:
                rl = rng.randint(0, L + 1)
            r = _row(rng, L, min(rl, L), V, end=rl < L)
            if rng.rand() < 0.4 and ln > 0:                         # copy a piece of the hypothesis: longer n-grams match
                a = rng.randint(0, min(ln, T))
                b = min(a + rng.randint(1, 6), min(ln, T), L)
                r[a:b] = h[a:b]
            refs.append(r)
        add(h, refs)
    hyp = np.stack(hyps)
    offs = np.concatenate([[0], np.cumsum([len(r) for r in ref_sets])]).astype(np.int32)
    refs = np.concatenate(ref_sets, 0)
    bleu = _bleu(ref_sets, hyps)
    return {'syn_hyp': hyp, 'syn_refs': refs.astype(np.int32), 'syn_offsets': offs, 'syn_bleu': bleu}


def gen_pascal():
    z = np.load(os.path.join(HERE, 'golden', 'ciderd_pascal.npz'))
    refs, cands = z['refs'].astype(np.int64), z['cands'].astype(np.int64)
    return {'pascal_bleu': _bleu([refs[i] for i in range(refs.shape[0])], [cands[i] for i in range(cands.shape[0])])}


def gen_full(scratch):
    from captioning.utils import rewards as R
    V, B, n, T = 30, 10, 5, 20
    df, ref_len = cdo.build_document_frequency(cdo.make_refs(300, V, seed=13))
    dd = defaultdict(float)
    dd.update({tuple(str(t) for t in k): v for k, v in df.items()})
    with open(os.path.join(scratch, 'data', 'bleu-df.p'), 'wb') as f:
        pickle.dump({'document_frequency': dd, 'ref_len': ref_len}, f, protocol=2)
    R.CiderD_scorer = None
    R.init_scorer('bleu-df')
    gts = cdo.make_refs(B, V, seed=17, L=T)
    rng = np.random.RandomState(5)

    def rows(k):
        out = np.zeros((k, T), np.int64)
        for i in range(k):
            ln = rng.randint(1, T + 1)
            out[i, :ln] = np.minimum(rng.zipf(1.3, size=ln), V)
        return out
    sampled, greedy = rows(B * n), rows(B)
    for i in range(B):                                              # pieces of the references: non-trivial scores
        sampled[i * n, :7] = gts[i][0][:7]
        sampled[i * n + 1, :10] = gts[i][2][:10]
        greedy[i, :5] = gts[i][1][:5]
    sampled[3] = 0
    res = {'full_gts': np.stack(gts), 'full_sampled': sampled, 'full_greedy': greedy, 'full_weights': np.array(WEIGHTS),
           'full_df_keys': np.array([list(k) + [-1] * (4 - len(k)) for k in df], np.int64), 'full_df_vals': np.array(list(df.values()), np.float64),
           'full_ref_len': np.array(float(ref_len)), 'full_meta': np.array([V, B, n, T])}
    for j, (wc, wb) in enumerate(WEIGHTS):
        opt = argparse.Namespace(cider_reward_weight=wc, bleu_reward_weight=wb)
        res['full_reward_%d' % j] = np.asarray(R.get_self_critical_reward(torch.from_numpy(greedy), gts, torch.from_numpy(sampled), opt), np.float64)
        res['full_scores_%d' % j] = np.asarray(R.get_scores(gts, torch.from_numpy(sampled), opt), np.float64) * np.ones(B * n)
    R.CiderD_scorer = None
    return res


def main():
    out = os.path.join(HERE, 'golden', 'bleu_reward.npz')
    scratch = _enter_scratch()
    rng = np.random.RandomState(2024)
    res = {}
    res.update(gen_synthetic(rng))
    res.update(gen_pascal())
    res.update(gen_full(scratch))
    np.savez_compressed(out, **res)
    print('bleu_reward: %d synthetic pairs (mean BLEU-4 %.4f), %d PASCAL-50S candidates (mean %.4f), %d weight pairs' %
          (len(res['syn_bleu']), res['syn_bleu'].mean(), len(res['pascal_bleu']), res['pascal_bleu'].mean(), len(WEIGHTS)))


if __name__ == '__main__':
    main()
