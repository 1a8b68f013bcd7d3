"""Generate tests/golden/coco_eval.npz from the LIVE coco-caption scorers of the reference checkout (build container only).

    python tests/make_coco_eval_golden.py        # needs the reference checkout that oracle/make_golden.py reads

Each caption is the string of its ids before the first 0 joined by single spaces, each reference the same of one 0-padded label row; the
unmodified Bleu(4), Rouge() and Cider() of coco-caption/pycocoevalcap score them, one compute_score call per round (caption j of every
image).  Cases (key prefix):
  small    per_image 1, T = L = 12: empty captions, an empty reference, a caption equal to a reference, repeated n-grams (clipping), ties
           for the closest reference length, 1 and 20 references, n-grams found in no reference, a caption without a closing 0
  long     per_image 1, T = L = 256: captions and references of 256 tokens
  split    per_image 1, 5000 images x 5 references of 8-16 tokens, T = 16
  oracle   per_image 5, 60 images x 5 references, T = 16
For each: <c>_seq [S, T] and <c>_refs [n_refs, L] int32 with <c>_nrefs [images] (the inputs), <c>_per, and the scorers' outputs
  <c>_bleu [S, 4]       per-sentence BLEU-1..4 (the second value of Bleu.compute_score, caption j of image i in row i * per + j)
  <c>_rouge [S], <c>_cider [S]
  <c>_overall [per, 6]  each round's Bleu_1..4 (corpus), ROUGE_L and CIDEr as compute_score returns them
and for the oracle case <c>_oracle [6] / <c>_avg [6]: eval_multi.eval_oracle's overall oracle_ / avg_ values of the six metrics.
"""
from __future__ import annotations

import contextlib
import io
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
sys.path.insert(0, REPO)

from oracle.make_golden import _enter_scratch                    # noqa: E402


def text(row):
    out = []
    for v in row:
        if int(v) == 0:
            break
        out.append(str(int(v)))
    return ' '.join(out)


def row(rng, T, lo, hi, vocab):
    r = np.zeros(T, np.int32)
    ln = rng.randint(lo, hi + 1)
    r[:ln] = rng.choice(vocab, size=ln)
    return r


def small_case(rng):
    T = 12
    common = np.arange(1, 20)
    seqs, refs = [], []
    def img(cap, rs):
        seqs.append(np.asarray(cap, np.int32))
        refs.append(np.stack([np.asarray(r, np.int32) for r in rs]))
    z = lambda ids: np.array(list(ids) + [0] * (T - len(ids)), np.int32)
    img(z([]), [row(rng, T, 3, 10, common) for _ in range(3)])                                      # empty caption
    img(z([]), [z([]), row(rng, T, 3, 10, common)])                                                # empty caption and an empty reference
    r = row(rng, T, 6, 10, common)
    img(r.copy(), [row(rng, T, 3, 10, common), r, row(rng, T, 3, 10, common)])                    # equal to a reference
    img(z([5, 5, 5, 5, 6, 6, 5, 5]), [z([5, 5, 7, 6, 5]), z([5, 6, 6, 5, 5, 8])])                  # repeated n-grams: clipping
    img(z([3, 4, 5, 6, 7, 8]), [z([3, 4, 5, 9, 9]), z([4, 5, 6, 7, 8, 2, 2]), z([1] * 9)])         # closest length: 5 and 7 tie
    img(z([2, 3, 4, 5]), [z([2, 3, 4, 9, 9, 9]), z([2, 3])])                                       # lengths 6 and 2 tie, longer first
    img(row(rng, T, 4, 10, common), [row(rng, T, 4, 10, common)])                                  # one reference
    img(row(rng, T, 4, 10, common), [row(rng, T, 2, 11, common) for _ in range(20)])               # twenty references
    img(z([25, 26, 27, 28, 29]), [row(rng, T, 4, 10, common) for _ in range(4)])                   # n-grams in no reference
    img(rng.choice(common, size=T).astype(np.int32), [row(rng, T, 6, T, common) for _ in range(5)])   # no closing 0
    for _ in range(6):
        img(row(rng, T, 1, T, common), [row(rng, T, 1, T, common) for _ in range(rng.randint(2, 7))])
    return np.stack(seqs), refs, 1


def long_case(rng):
    T, vocab = 256, np.arange(1, 40)
    seqs, refs = [], []
    for i in range(4):
        seqs.append(rng.choice(vocab, size=T).astype(np.int32) if i % 2 == 0 else row(rng, T, 180, 255, vocab))
        rs = [rng.choice(vocab, size=T).astype(np.int32), row(rng, T, 150, 255, vocab), row(rng, T, 10, 60, vocab)]
        rs[1][:100] = seqs[-1][:100]
        refs.append(np.stack(rs))
    return np.stack(seqs), refs, 1


def pooled_case(rng, B, per, T=16, V=9487):
    seqs, refs = np.zeros((B * per, T), np.int32), []
    for i in range(B):
        pool = rng.randint(1, V + 1, size=20)
        for j in range(per):
            seqs[i * per + j] = row(rng, T, 8, 16, pool)
        refs.append(np.stack([row(rng, T, 8, 16, pool) for _ in range(5)]))
    return seqs, refs, per


def score(seqs, refs, per):
    from pycocoevalcap.bleu.bleu import Bleu
    from pycocoevalcap.rouge.rouge import Rouge
    from pycocoevalcap.cider.cider import Cider
    B = len(refs)
    gts = {i: [text(r) for r in refs[i]] for i in range(B)}
    S = B * per
    bleu, rouge, cider, overall = np.zeros((S, 4)), np.zeros(S), np.zeros(S), np.zeros((per, 6))
    for j in range(per):
        res = {i: [text(seqs[i * per + j])] for i in range(B)}
        with contextlib.redirect_stdout(io.StringIO()):            # Bleu prints its totals
            b, bs = Bleu(4).compute_score(gts, res)
        r, rs = Rouge().compute_score(gts, res)
        c, cs = Cider().compute_score(gts, res)
        bleu[j::per] = np.array(bs).T
        rouge[j::per], cider[j::per] = rs, cs
        overall[j] = list(b) + [r, c]
    return bleu, rouge, cider, overall


def main():
    out_path = os.path.join(HERE, 'golden', 'coco_eval.npz')
    d = _enter_scratch()
    sys.path.insert(0, os.path.join(d, 'coco-caption'))
    rng = np.random.RandomState(2026)
    res = {}
    for name, (seqs, refs, per) in (('small', small_case(rng)), ('long', long_case(rng)), ('split', pooled_case(rng, 5000, 1)),
                                    ('oracle', pooled_case(rng, 60, 5))):
        bleu, rouge, cider, overall = score(seqs, refs, per)
        res.update({name + '_seq': seqs, name + '_refs': np.concatenate(refs), name + '_nrefs': np.array([len(r) for r in refs], np.int32),
                    name + '_per': np.array(per), name + '_bleu': bleu, name + '_rouge': rouge, name + '_cider': cider,
                    name + '_overall': overall})
        if per > 1:                                                  # eval_multi.py:104-117 over the rounds' per-image scores
            B = len(refs)
            m = np.concatenate([bleu, rouge[:, None], cider[:, None]], 1).reshape(B, per, 6)
            res[name + '_oracle'] = np.array([np.array([max(m[i, :, k].tolist()) for i in range(B)]).mean() for k in range(6)])
            res[name + '_avg'] = np.array([np.array([sum(m[i, :, k].tolist()) / per for i in range(B)]).mean() for k in range(6)])
        print('%s: %d captions, overall %s' % (name, len(seqs), np.round(overall[0], 4)))
    np.savez_compressed(out_path, **res)


if __name__ == '__main__':
    main()
