"""CPU restatement of the BLEU-4 reward term and of the weighted reward -- the checker of the device kernels (test infrastructure only).

Reference lines followed (paths relative to the reference checkout):
  tokens_through_eos    captioning/utils/rewards.py:33-39 (array_to_str: tokens through the first 0, the 0 a word of its own)
  bleu4                 coco-caption/pycocoevalcap/bleu/bleu_scorer.py:26-80 (precook, cook_refs, cook_test) and :184-260
                        (compute_score(option='closest'): the per-sentence bleu_list[3])
  weighted_scores       captioning/utils/rewards.py:63-74 and :100-112 (a term only when its weight is > 0, combined in float64)
  self_critical_reward  captioning/utils/rewards.py:76-81 (score(sample) - score(greedy of its image), then float32 in LossWrapper)
  loo_reward            captioning/modules/losses.py:61-62,168-187 (scores cast to float32, then the leave-one-out baseline)
Pinned by tests/golden/bleu_reward.npz, which tests/make_bleu_golden.py wrote from the live reference scorer.
"""
from __future__ import annotations

import math
from collections import Counter
from typing import Sequence

import numpy as np

from oracle import ciderd_oracle as cdo

tokens_through_eos = cdo.tokens_through_eos


def _counts(tokens, n):
    return Counter(tuple(tokens[i:i + n]) for i in range(len(tokens) - n + 1))


def bleu4(hyp: Sequence[int], refs: Sequence[Sequence[int]]) -> float:
    """Per-sentence BLEU-4 of one hypothesis (token list, already cut through the first 0) against token lists."""
    assert len(refs) >= 1
    testlen = len(hyp)
    reflen = min((abs(len(r) - testlen), len(r)) for r in refs)[1]
    bleu = 1.0
    for k in range(4):
        hc = _counts(hyp, k + 1)
        ref_max = Counter()
        for r in refs:
            for g, c in _counts(r, k + 1).items():
                ref_max[g] = max(ref_max[g], c)
        correct = sum(min(c, ref_max.get(g, 0)) for g, c in hc.items())
        guess = max(0, testlen - k)
        bleu *= (float(correct) + 1e-15) / (float(guess) + 1e-9)
    score = bleu ** (1. / 4)
    ratio = (testlen + 1e-15) / (reflen + 1e-9)
    if ratio < 1:
        score *= math.exp(1 - 1 / ratio)
    return score


def bleu_scores(hyp_rows: np.ndarray, ref_rows_per_hyp: Sequence[np.ndarray]) -> np.ndarray:
    """BLEU-4 of every hypothesis row against its own reference rows (all cut through the first 0)."""
    return np.array([bleu4(tokens_through_eos(h), [tokens_through_eos(r) for r in refs]) for h, refs in zip(hyp_rows, ref_rows_per_hyp)])


def weighted_scores(hyp_rows: np.ndarray, ref_rows_per_hyp, weights, df=None, ref_len=None) -> np.ndarray:
    """cider_weight * CIDEr-D + bleu_weight * BLEU-4 per hypothesis; a term is computed only when its weight is > 0, else it is 0."""
    wc, wb = (float(w) for w in weights)
    if wc > 0:
        cider = cdo.ciderd_scores([tokens_through_eos(h) for h in hyp_rows], [[tokens_through_eos(r) for r in refs] for refs in ref_rows_per_hyp],
                                  df, ref_len)
    else:
        cider = 0
    bleu = bleu_scores(hyp_rows, ref_rows_per_hyp) if wb > 0 else 0
    return np.asarray(wc * cider + wb * bleu, dtype=np.float64) * np.ones(len(hyp_rows))


def self_critical_reward(greedy: np.ndarray, gts: Sequence[np.ndarray], sampled: np.ndarray, weights, df=None, ref_len=None):
    """(reward float64 [S, T], scores float64 [S + B]) of get_self_critical_reward with both terms."""
    B, S = len(gts), sampled.shape[0]
    n = S // B
    hyps = np.concatenate([sampled, greedy], 0)
    refs = [gts[i // n] for i in range(S)] + [gts[i] for i in range(B)]
    scores = weighted_scores(hyps, refs, weights, df, ref_len)
    diff = scores[:S].reshape(B, n) - scores[-B:][:, None]
    return np.repeat(diff.reshape(S)[:, None], sampled.shape[1], 1), scores


def get_scores(gts: Sequence[np.ndarray], sampled: np.ndarray, weights, df=None, ref_len=None) -> np.ndarray:
    """get_scores with both terms: float64 [S]."""
    n = sampled.shape[0] // len(gts)
    return weighted_scores(sampled, [gts[i // n] for i in range(sampled.shape[0])], weights, df, ref_len)


def loo_reward(scores: np.ndarray, n: int) -> np.ndarray:
    """new_self_critical's per-row reward [S] (float32): the scores cast to float32 first, then minus the mean of the image's other samples."""
    s = scores.astype(np.float32).reshape(-1, n)
    return (s - (s.sum(1, keepdims=True) - s) / np.float32(n - 1)).reshape(-1)
