"""Captions and references past 64 tokens on the host side: the float64 restatements the GPU tests check against (oracle/ciderd_oracle.py,
tests/bleu_oracle.py) reproduce the reference's own CiderD and Bleu scorers on 65-, 100- and 256-token rows (tests/golden/long_captions.npz,
made by tests/make_long_captions_golden.py); the Python surface takes max_length 256 on every family up to the device; the diversity
functions keep their 64-token limit."""
import argparse
import os
import re

import numpy as np
import pytest
import torch

from helpers import REPO, co, family_opt
import bleu_oracle as bo
from oracle import ciderd_oracle as cdo

GOLD = os.path.join(REPO, 'tests', 'golden', 'long_captions.npz')


def load_case():
    g = np.load(GOLD)
    V, B, n, T, L = (int(x) for x in g['meta'])
    gts = [g['gts'][i][:int(g['ref_counts'][i])] for i in range(B)]
    df = {tuple(int(t) for t in k if t >= 0): float(v) for k, v in zip(g['df_keys'], g['df_vals'])}
    return g, gts, df, float(g['ref_len']), n


def corpus_df(gts, entries_per_image):
    df, images = cdo.build_document_frequency(gts)
    return {k: v * entries_per_image for k, v in df.items()}, images * entries_per_image


def test_golden_covers_long_rows():
    g, gts, _, _, n = load_case()
    hyp_len = [len(cdo.tokens_through_eos(r)) for r in np.concatenate([g['sampled'], g['greedy']])]
    ref_len = [len(cdo.tokens_through_eos(r)) for rows in gts for r in rows]
    assert {66, 101, 256} <= set(hyp_len) and {66, 101, 256} <= set(ref_len)        # words + the closing 0; 256 words and no 0
    assert min(len(cdo.tokens_through_eos(r)) for r in gts[1]) < 16 and max(len(cdo.tokens_through_eos(r)) for r in gts[1]) > 200
    assert (g['scores_0'] > 0.3).sum() >= 4 and (g['bleu'] > 0.5).sum() >= 4


def test_restatement_reproduces_reference_bleu():
    g, gts, _, _, n = load_case()
    hyps = np.concatenate([g['sampled'], g['greedy']])
    refs = [gts[i // n] for i in range(len(g['sampled']))] + gts
    got = bo.bleu_scores(hyps, refs)
    assert np.abs(got - g['bleu']).max() < 1e-15


@pytest.mark.parametrize('table', ['pickle', 'corpus'])
def test_restatement_reproduces_reference_rewards(table):
    g, gts, df, ref_len, n = load_case()
    pre = '' if table == 'pickle' else 'c'
    for j, w in enumerate(np.asarray(g['weights'])):
        if table == 'corpus':
            df, ref_len = corpus_df(gts, n + 1)
        reward, _ = bo.self_critical_reward(g['greedy'], gts, g['sampled'], tuple(w), df, ref_len)
        assert np.abs(reward - g['%sreward_%d' % (pre, j)]).max() < 1e-12, (table, j)
        if table == 'corpus':
            df, ref_len = corpus_df(gts, n)
        scores = bo.get_scores(gts, g['sampled'], tuple(w), df, ref_len)
        assert np.abs(scores - g['%sscores_%d' % (pre, j)]).max() < 1e-12, (table, j)


def test_restatement_keeps_the_length_penalty_past_64():
    """CIDEr-D's Gaussian length penalty (sigma 6, on bigram counts) applies at any length: a 200-token hypothesis that copies a 256-token
    reference's first 200 tokens scores below the copy of the whole reference."""
    _, gts, df, ref_len, _ = load_case()
    ref = gts[0][2]
    whole = cdo.ciderd_scores([cdo.tokens_through_eos(ref)], [[cdo.tokens_through_eos(ref)]], df, ref_len)[0]
    part = cdo.ciderd_scores([list(ref[:200]) + [0]], [[cdo.tokens_through_eos(ref)]], df, ref_len)[0]
    assert whole > 1.0 and 0.0 < part < whole * np.exp(-(55 ** 2) / 72.0) * 1.01


@pytest.mark.parametrize('family', ['updown', 'att2in2', 'newfc', 'transformer', 'aoa'])
def test_every_family_takes_max_length_256(family):
    """Nothing on the Python side refuses a 256-token max_length: greedy, sampling and beam decoding stop at the no-CPU-tensor check."""
    import imagecaptioning.pytorch_b200 as b200
    cfg = dict(V=30, E=16, H=16, A=8, F_fc=16, F_att=16, T=256)
    if family == 'transformer':
        cfg = dict(cfg, E=16, H=32, A=1)
    model = b200.setup(family_opt(family, heads=2, **cfg))
    assert model.seq_length == 256
    fc, att = co.make_inputs(2, 3, 16, 16, seed=1)
    for opt in ({'sample_method': 'greedy', 'beam_size': 1}, {'sample_method': 'sample', 'beam_size': 1, 'sample_n': 2},
                {'beam_size': 5, 'sample_n': 1}):
        with pytest.raises(RuntimeError, match='CUDA'):
            model(fc, att, None, opt=opt, mode='sample')


def test_rewards_take_256_token_rows_up_to_the_device():
    import imagecaptioning.pytorch_b200 as b200
    g, gts, _, _, n = load_case()
    b200.rewards.CiderD_scorer = object.__new__(b200.rewards.CiderDTable)
    try:
        opt = argparse.Namespace(cider_reward_weight=0.7, bleu_reward_weight=0.3)
        with pytest.raises(RuntimeError, match='CUDA'):
            b200.rewards.get_self_critical_reward(torch.from_numpy(g['greedy']), gts, torch.from_numpy(g['sampled']), opt)
        with pytest.raises(RuntimeError, match='CUDA'):
            b200.rewards.get_scores(gts, torch.from_numpy(g['sampled']), opt)
    finally:
        b200.rewards.CiderD_scorer = None


def test_diversity_stays_at_64_tokens(monkeypatch):
    import imagecaptioning.pytorch_b200 as b200

    def refuse(*a, **k):
        raise AssertionError('device work before the guard')
    monkeypatch.setattr(b200._lib, 'load', refuse)
    seqs = torch.ones(4, 65, dtype=torch.long)
    with pytest.raises(ValueError, match='between 1 and 64'):
        b200.eval_multi.div_stats(seqs, 2)
    with pytest.raises(ValueError, match='between 1 and 64'):
        b200.rewards.check_caption_sets(4, 2, 65)
    assert b200.rewards.check_caption_sets(4, 2, 64) == 2


def test_length_bound_documented_in_header():
    src = open(os.path.join(REPO, 'include', 'capb200.h')).read()
    assert re.search(r'#define CAPB200_MAX_SEQ_LENGTH 256\b', src)
    for name in ('capb200_tfm_dec_self_attention', 'capb200_mha_causal_forward', 'capb200_mha_causal_backward'):
        assert re.search(r'\bint %s\(' % name, src), name
