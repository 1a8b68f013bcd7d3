"""Float64 restatement of the reference's caption-set diversity scores over id rows (no strings, no dicts of words):

    self_cider_matrix / get_div   cider/pyciderevalcap/cider/cider_scorer.py:51-77,186-212,240-258, captioning/utils/rewards.py:116-138
    div_n / global_div_1          captioning/utils/div_utils.py:10-35
    mutual_bleu                   captioning/utils/eval_multi.py:140-152 over coco-caption's Bleu(4) (closest reference length)

A caption is its ids through the first 0 (``with_eos``, array_to_str) or before it (the decoded words).  Rows are n per image, image-major.
"""
from __future__ import annotations

import math
from collections import defaultdict
from typing import Dict, List, Sequence, Tuple

import numpy as np


def caption(row, with_eos: bool) -> List[int]:
    out = []
    for v in row:
        v = int(v)
        if v == 0:
            if with_eos:
                out.append(0)
            break
        out.append(v)
    return out


def ngram_counts(w: Sequence[int], n: int = 4) -> Dict[Tuple[int, ...], int]:
    counts: Dict[Tuple[int, ...], int] = {}
    for k in range(1, n + 1):
        for i in range(len(w) - k + 1):
            g = tuple(w[i:i + k])
            counts[g] = counts.get(g, 0) + 1
    return counts


def counts2vec(cnts, df, log_ref_len):
    vec = [dict() for _ in range(4)]
    norm = [0.0] * 4
    for g, tf in cnts.items():
        k = len(g) - 1
        vec[k][g] = float(tf) * (log_ref_len - np.log(max(1.0, df.get(g, 0.0))))
        norm[k] += vec[k][g] ** 2
    return vec, [np.sqrt(x) for x in norm]


def self_cider_matrix(caps: Sequence[Sequence[int]], df, ref_len: float) -> np.ndarray:
    """my_get_self_cider: 10 * mean over orders of the tf-idf cosine of every pair of captions; ref_len is the un-logged count."""
    log_ref_len = np.log(float(ref_len))
    vecs = [counts2vec(ngram_counts(c), df, log_ref_len) for c in caps]
    n = len(caps)
    m = np.zeros((n, n, 4))
    for i, (vi, ni) in enumerate(vecs):
        for j, (vj, nj) in enumerate(vecs):
            for k in range(4):
                v = 0.0
                for g, w in vi[k].items():
                    v += w * vj[k].get(g, 0.0)
                if ni[k] != 0 and nj[k] != 0:
                    v /= ni[k] * nj[k]
                m[i, j, k] = v
    return np.mean(m, -1) * 10.0


def get_div(mat: np.ndarray) -> float:
    with np.errstate(divide='ignore', invalid='ignore'):
        ev = np.clip(np.linalg.eigvalsh(mat / 10), 0, None)
        return float(-np.log(np.sqrt(ev[-1]) / np.sqrt(ev).sum()) / np.log(len(ev)))


def self_cider(seqs: np.ndarray, n: int, df, ref_len: float, with_eos: bool):
    B = seqs.shape[0] // n
    mats = np.stack([self_cider_matrix([caption(r, with_eos) for r in seqs[i * n:(i + 1) * n]], df, ref_len) for i in range(B)])
    return mats, np.array([get_div(m) for m in mats])


def div_n(seqs: np.ndarray, n: int, order: int) -> np.ndarray:
    B = seqs.shape[0] // n
    out = []
    for i in range(B):
        grams, total = set(), 0
        for r in seqs[i * n:(i + 1) * n]:
            w = caption(r, False)
            total += len(w)
            grams.update(tuple(w[p:p + order]) for p in range(len(w) - order + 1))
        out.append(float(len(grams)) / (1e-6 + float(total)))
    return np.array(out)


def global_div_1(seqs: np.ndarray) -> float:
    words = set()
    for r in seqs:
        words.update(caption(r, False))
    return float(len(words))


def bleu_stats(hyp: Sequence[int], refs: Sequence[Sequence[int]]):
    """(correct[4], guess[4], testlen, closest reflen) of one hypothesis (bleu_scorer.py cook_refs / cook_test)."""
    maxc: Dict[Tuple[int, ...], int] = {}
    for r in refs:
        for g, c in ngram_counts(r).items():
            maxc[g] = max(maxc.get(g, 0), c)
    correct = [0] * 4
    for g, c in ngram_counts(hyp).items():
        correct[len(g) - 1] += min(maxc.get(g, 0), c)
    tl = len(hyp)
    reflen = min((abs(len(r) - tl), len(r)) for r in refs)[1]
    return correct, [max(0, tl - k) for k in range(4)], tl, reflen


def bleu_from(correct, guess, testlen, reflen):
    tiny, small = 1e-15, 1e-9
    b, out = 1.0, []
    for k in range(4):
        b *= float(correct[k] + tiny) / (guess[k] + small)
        out.append(b ** (1.0 / (k + 1)))
    ratio = (testlen + tiny) / (reflen + small)
    if ratio < 1:
        out = [x * math.exp(1 - 1 / ratio) for x in out]
    return out


def mutual_bleu(seqs: np.ndarray, n: int):
    """(all_scrs [n, 4] corpus BLEU-1..4 per leave-one-out round, scrperimg [n, B] per-sentence BLEU-2)."""
    B = seqs.shape[0] // n
    caps = [[caption(r, False) for r in seqs[i * n:(i + 1) * n]] for i in range(B)]
    all_scrs, scrperimg = np.zeros((n, 4)), np.zeros((n, B))
    for j in range(n):
        tot_c, tot_g, tl, rl = [0] * 4, [0] * 4, 0, 0
        for i in range(B):
            c, g, t, r = bleu_stats(caps[i][j], caps[i][:j] + caps[i][j + 1:])
            tot_c = [a + b for a, b in zip(tot_c, c)]
            tot_g = [a + b for a, b in zip(tot_g, g)]
            tl, rl = tl + t, rl + r
            scrperimg[j, i] = bleu_from(c, g, t, r)[1]
        all_scrs[j] = bleu_from(tot_c, tot_g, tl, rl)
    return all_scrs, scrperimg


def document_frequency(refs_per_image, with_eos: bool):
    df: Dict[Tuple[int, ...], float] = defaultdict(float)
    for rows in refs_per_image:
        seen = set()
        for r in rows:
            seen.update(ngram_counts(caption(r, with_eos)).keys())
        for g in seen:
            df[g] += 1.0
    return dict(df), len(refs_per_image)
