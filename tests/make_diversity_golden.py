"""Generate tests/golden/diversity.npz from the LIVE reference (build container only; the reference checkout is read-only).

    python tests/make_diversity_golden.py        # needs the reference checkout that oracle/make_golden.py reads

For n = 2, 5, 10 and 32 captions per image (V = 9487, T = 16; seeded random ids, repeated captions, an image whose captions are all the
same, empty captions -- 0 at position 0 -- and captions without a closing 0) the file holds, keyed by n:
  seqs_<n> [B*n, T], refs_<n> [B, 5, T]                          the caption sets and the references the document frequencies come from
  rscore_<n> [B]                                                  the unmodified rewards.get_self_cider_scores, after init_scorer reads a
                                                                  pickle df of the references written into the scratch data/ (a defaultdict,
                                                                  so that an unseen n-gram has df 0 instead of raising KeyError)
  rmat_<n> [B, n, n]                                              Cider_scorer.my_self_cider on the same array_to_str captions
  dfk_<n> [m, 4], dfv_<n> [m], ref_len_<n>                       that pickle's df (keys padded with -1) and ref_len
  emat_<n>, escore_<n>, eself_<n>                                 eval_self_cider's matrices, scores and overall score on 'w<id>' words: the
                                                                  same Cider(df='corpus') + compute_doc_freq + ref_len = log(images) steps
  div1_<n>, div2_<n>, gdiv1_<n>, adiv1_<n> [B], adiv2_<n> [B]   compute_div_n / compute_global_div_n on those words
  mbleu_<n> [n, 4], scrperimg_<n> [n, B]                          eval_div_stats' Bleu(4) leave-one-out rounds
The Java PTB tokenizer is skipped: 'w<id>' words pass through it unchanged.
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

from oracle.make_golden import _enter_scratch                    # noqa: E402

V, T, N_REFS = 9487, 16, 5
CASES = {2: 8, 5: 9, 10: 6, 32: 4}           # n -> images


def array_to_str(arr):
    out = ''
    for v in arr:
        out += str(int(v)) + ' '
        if v == 0:
            break
    return out.strip()


def words(arr):
    out = []
    for v in arr:
        if v == 0:
            break
        out.append('w%d' % int(v))
    return ' '.join(out)


def make_set(n, B, rng):
    seqs = np.zeros((B * n, T), np.int64)
    refs = np.zeros((B, N_REFS, T), np.int64)
    for i in range(B):
        pool = rng.randint(1, V + 1, size=8)
        pool[0] = V                                                  # the largest id
        def row(lo=0):
            ln = rng.randint(lo, T + 1)
            r = np.zeros(T, np.int64)
            toks = np.where(rng.rand(ln) < 0.7, pool[rng.randint(0, 8, size=ln)], rng.randint(1, V + 1, size=ln))
            r[:ln] = toks
            return r
        for j in range(n):
            seqs[i * n + j] = row()
        for j in range(N_REFS):
            refs[i, j] = row(lo=1)
        if i % 3 == 1:
            seqs[i * n + 1] = seqs[i * n]                            # a repeated caption
        if i == 2:
            seqs[i * n:(i + 1) * n] = seqs[i * n]                    # every caption the same
        if i == 0:
            seqs[i * n] = 0                                          # an empty caption
            seqs[i * n + n - 1, :] = pool[rng.randint(0, 8, size=T)]   # no closing 0
        if i == 3 and n == 5:
            seqs[i * n:(i + 1) * n] = 0                              # every caption empty
        refs[i, 0, :4] = seqs[i * n + n - 1, :4]                     # shared n-grams with the references
    return seqs, refs


def main():
    out_path = os.path.join(HERE, 'golden', 'diversity.npz')
    d = _enter_scratch()
    from captioning.utils import rewards as R
    from captioning.utils import div_utils
    from pyciderevalcap.cider.cider import Cider
    from pycocoevalcap.bleu.bleu import Bleu
    rng = np.random.RandomState(2024)
    res = {'meta': np.array([V, T, N_REFS])}
    for n, B in CASES.items():
        seqs, refs = make_set(n, B, rng)
        # --- reward form: a prepro_ngrams-style pickle of the references (array_to_str keeps the 0), read by init_scorer
        df = defaultdict(float)
        for i in range(B):
            seen = set()
            for r in refs[i]:
                w = array_to_str(r).split()
                for k in range(1, 5):
                    for p in range(len(w) - k + 1):
                        seen.add(tuple(w[p:p + k]))
            for g in seen:
                df[g] += 1.0
        name = 'div%d' % n
        with open(os.path.join(d, 'data', name + '.p'), 'wb') as f:
            pickle.dump({'document_frequency': df, 'ref_len': B}, f)
        R.CiderD_scorer = R.Cider_scorer = R.Bleu_scorer = None
        R.init_scorer(name)
        gts = [refs[i] for i in range(B)]
        res['rscore_%d' % n] = np.asarray(R.get_self_cider_scores(gts, torch.from_numpy(seqs), argparse.Namespace()), np.float64)
        res['rmat_%d' % n] = np.stack(R.Cider_scorer.my_self_cider([[array_to_str(r) for r in seqs[i * n:(i + 1) * n]] for i in range(B)]))
        keys = list(df.keys())
        dfk = np.full((len(keys), 4), -1, np.int32)
        for m, g in enumerate(keys):
            dfk[m, :len(g)] = [int(t) for t in g]
        res['dfk_%d' % n], res['dfv_%d' % n], res['ref_len_%d' % n] = dfk, np.array([df[g] for g in keys]), np.array(float(B))
        # --- eval_self_cider on words (eval_multi.py:177-217 without the tokenizer)
        scorer = Cider(df='corpus')
        for i in range(B):
            scorer.cider_scorer += (None, [words(r) for r in refs[i]])
        scorer.cider_scorer.compute_doc_freq()
        scorer.cider_scorer.ref_len = np.log(float(len(scorer.cider_scorer.crefs)))
        caps = {i: [words(r) for r in seqs[i * n:(i + 1) * n]] for i in range(B)}
        mats = scorer.my_self_cider([caps[i] for i in range(B)])

        def get_div(eigvals):
            eigvals = np.clip(eigvals, 0, None)
            return -np.log(np.sqrt(eigvals[-1]) / (np.sqrt(eigvals).sum())) / np.log(len(eigvals))
        with np.errstate(divide='ignore', invalid='ignore'):
            sc = [get_div(np.linalg.eigvalsh(m / 10)) for m in mats]
        res['emat_%d' % n], res['escore_%d' % n], res['eself_%d' % n] = np.stack(mats), np.array(sc), np.array(np.mean(np.array(sc)))
        # --- eval_div_stats (eval_multi.py:121-175 without the tokenizer)
        div_1, adiv_1 = div_utils.compute_div_n(caps, 1)
        div_2, adiv_2 = div_utils.compute_div_n(caps, 2)
        globdiv_1, _ = div_utils.compute_global_div_n(caps, 1)
        bleu = Bleu(4)
        all_scrs, scrperimg = [], np.zeros((n, B))
        for j in range(n):
            temp_refs = {k: caps[k][:j] + caps[k][j + 1:] for k in caps}
            cands = {k: [caps[k][j]] for k in caps}
            score, scores = bleu.compute_score(temp_refs, cands)
            all_scrs.append(score)
            scrperimg[j, :] = scores[1]
        res.update({'div1_%d' % n: np.array(div_1), 'div2_%d' % n: np.array(div_2), 'gdiv1_%d' % n: np.array(globdiv_1),
                    'adiv1_%d' % n: adiv_1, 'adiv2_%d' % n: adiv_2, 'mbleu_%d' % n: np.array(all_scrs), 'scrperimg_%d' % n: scrperimg,
                    'seqs_%d' % n: seqs, 'refs_%d' % n: refs})
        print('n=%d: %d images, self-CIDEr %s, Div1 %.4f, mBLEU-4 %.4f' % (n, B, np.round(res['rscore_%d' % n], 4), div_1, np.mean(all_scrs, 0)[3]))
    np.savez_compressed(out_path, **res)


if __name__ == '__main__':
    main()
