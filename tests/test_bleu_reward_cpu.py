"""The BLEU-4 reward term and the reward weights on the host side: the numpy restatement (bleu_oracle) against the live-reference goldens of
tests/make_bleu_golden.py, the ctypes mirrors against include/capb200.h, and B200LossWrapper's dispatch of non-default weights to the fused
steps (entropy and self-CIDEr rewards stay refused)."""
import argparse
import os
import re

import numpy as np
import pytest
import torch

from helpers import REPO, family_opt
import bleu_oracle as bo

GOLD = os.path.join(REPO, 'tests', 'golden', 'bleu_reward.npz')


def full_case(g):
    V, B, n, T = (int(x) for x in g['full_meta'])
    df = {tuple(int(t) for t in k if t >= 0): float(v) for k, v in zip(g['full_df_keys'], g['full_df_vals'])}
    gts = [g['full_gts'][i] for i in range(B)]
    return gts, g['full_sampled'], g['full_greedy'], df, float(g['full_ref_len']), n


def syn_refs(g, i):
    return g['syn_refs'][g['syn_offsets'][i]:g['syn_offsets'][i + 1]]


def test_restatement_reproduces_synthetic_bleu():
    g = np.load(GOLD)
    got = np.array([bo.bleu4(bo.tokens_through_eos(h), [bo.tokens_through_eos(r) for r in syn_refs(g, i)]) for i, h in enumerate(g['syn_hyp'])])
    assert np.abs(got - g['syn_bleu']).max() < 1e-15
    # the golden covers what it claims to: a "0"-only hypothesis, rows without a 0, 1 and >= 5 references, positive and ~zero scores
    assert any(not h.any() for h in g['syn_hyp']) and any(h.all() for h in g['syn_hyp'])
    counts = np.diff(g['syn_offsets'])
    assert counts.min() == 1 and (counts >= 5).any() and counts.max() > 32
    assert (g['syn_bleu'] > 0.5).sum() > 10 and (g['syn_bleu'] < 1e-3).sum() > 10


def test_restatement_closest_length_tie_takes_the_shorter():
    """hypothesis "1 2 3 4 0" (5 words) against references of 4 and 6 words: reflen 4, no brevity penalty."""
    hyp = [1, 2, 3, 4, 0]
    short_first = bo.bleu4(hyp, [[1, 2, 3, 0], [1, 2, 3, 4, 5, 0]])
    long_first = bo.bleu4(hyp, [[1, 2, 3, 4, 5, 0], [1, 2, 3, 0]])
    assert short_first == long_first
    g = np.load(GOLD)
    assert abs(short_first - float(g['syn_bleu'][4])) < 1e-15


def test_restatement_reproduces_pascal_bleu():
    g = np.load(GOLD)
    z = np.load(os.path.join(REPO, 'tests', 'golden', 'ciderd_pascal.npz'))
    refs, cands = z['refs'].astype(np.int64), z['cands'].astype(np.int64)
    got = bo.bleu_scores(cands, [refs[i] for i in range(refs.shape[0])])
    assert np.abs(got - g['pascal_bleu']).max() < 1e-15
    assert g['pascal_bleu'].mean() > 0.1


def test_restatement_reproduces_weighted_rewards():
    g = np.load(GOLD)
    gts, sampled, greedy, df, ref_len, n = full_case(g)
    for j, w in enumerate(g['full_weights']):
        reward, _ = bo.self_critical_reward(greedy, gts, sampled, w, df, ref_len)
        assert np.abs(reward - g['full_reward_%d' % j]).max() < 1e-12, w
        scores = bo.get_scores(gts, sampled, w, df, ref_len)
        assert np.abs(scores - g['full_scores_%d' % j]).max() < 1e-12, w
        assert np.abs(g['full_reward_%d' % j]).max() > 1e-3
    # a weight <= 0 switches its term off instead of subtracting it: (-1, 1) scores BLEU-4 alone
    assert np.array_equal(g['full_scores_4'], g['full_scores_1'])


def test_ctypes_mirrors_match_header():
    import imagecaptioning.pytorch_b200 as b200
    L = b200._lib
    hdr = open(os.path.join(REPO, 'include', 'capb200.h')).read()
    body = re.search(r'typedef struct \{([^}]*)\} capb200_reward_weights;', hdr).group(1)
    assert re.findall(r'double\s+(\w+);', body) == ['cider', 'bleu'] == [f for f, _ in L.RewardWeights._fields_]
    for cname, py in (('capb200_scst_opts', L.ScstOpts), ('capb200_aoa_scst_opts', L.AoaScstOpts), ('capb200_tfm_scst_opts', L.TfmScstOpts)):
        body = re.search(r'typedef struct \{([^{}]*)\} %s;' % cname, hdr).group(1)
        body = re.sub(r'/\*.*?\*/', '', body, flags=re.S)
        fields = [f for decl in body.split(';') if decl.strip() for f in re.findall(r'(\w+)\s*(?:,|$)', decl.strip())]
        assert fields == [f for f, _ in py._fields_], cname
        assert py._fields_[-1] == ('reward_weights', __import__('ctypes').POINTER(L.RewardWeights))
        assert not py().reward_weights                  # a zero-initialised struct carries NULL: the CIDEr-D reward
    for name in ('capb200_bleu4_scores', 'capb200_weighted_reward'):
        decl = re.search(r'int %s\(([^)]*)\);' % name, hdr).group(1)
        assert len(decl.split(',')) == len(L.SIGNATURES[name][1]), name


def test_reference_list_refused_before_device_work():
    import imagecaptioning.pytorch_b200 as b200
    gts = [np.ones((2, 5), np.int64), np.zeros((0, 5), np.int64)]
    with pytest.raises(ValueError, match='reference'):
        b200.rewards.weights_struct((0.5, 0.5), gts)
    with pytest.raises(ValueError, match='reference'):
        b200.rewards.bleu_scores(gts, torch.zeros(2, 5, dtype=torch.long))
    assert b200.rewards.weights_struct((1.0, 0.0), gts).bleu == 0.0       # without the BLEU term the CIDEr-D path decides, as before
    assert b200.rewards.weights_struct(None, gts) is None
    with pytest.raises(ValueError, match='finite'):
        b200.rewards.weights_struct((float('nan'), 1.0), gts[:1])


def _wrapper_opt(**kw):
    opt = dict(sc_sample_method='greedy', sc_beam_size=1, train_sample_method='sample', train_beam_size=1, train_sample_n=5, cider_reward_weight=1,
               bleu_reward_weight=0, structure_loss_type='new_self_critical', structure_loss_weight=1.0, label_smoothing=0.0, use_ppo=0)
    opt.update(kw)
    return argparse.Namespace(**opt)


def _newfc():
    import imagecaptioning.pytorch_b200 as b200
    m = b200.setup(family_opt('newfc', 30, 16, 16, 8, 16, 16, 5)).train()
    B = 2
    fc, att = torch.zeros(B, 16), torch.zeros(B, 0, 0)
    labels, masks = torch.zeros(B, 5, 7, dtype=torch.long), torch.ones(B, 5, 7)
    labels[:, :, 1] = 3
    return b200, m, fc, att, labels, masks, [np.ones((1, 5), np.int64)] * B


@pytest.mark.skipif(torch.cuda.is_available(), reason='checks the behaviour of a box without a GPU')
@pytest.mark.parametrize('branch', ['sc', 'struc'])
@pytest.mark.parametrize('weights', [(0.7, 0.3), (0.0, 1.0), (2.0, 0.0)])
def test_loss_wrapper_dispatches_weighted_reward_to_fused_steps(branch, weights):
    """Non-default reward weights reach the fused steps (no NotImplementedError); the call stops at the engine's refusal of CPU tensors,
    and the step is handed the weights."""
    b200, m, fc, att, labels, masks, gts = _newfc()
    seen = {}
    step = m.scst_step

    def spy(*a, **kw):
        seen['w'] = kw.get('reward_weights')
        return step(*a, **kw)
    m.scst_step = spy
    lw = b200.B200LossWrapper(m, _wrapper_opt(cider_reward_weight=weights[0], bleu_reward_weight=weights[1]))
    lw._scorer = lambda: None           # the CIDEr-D table lives on a GPU; the step refuses the CPU tensors before it would read it
    with pytest.raises(RuntimeError, match='CUDA'):
        lw(fc, att, labels, masks, None, gts, torch.arange(2), branch == 'sc', branch == 'struc', False)
    assert seen['w'] == weights


@pytest.mark.parametrize('which', ['entropy_reward_weight', 'self_cider_reward_weight'])
def test_entropy_and_self_cider_rewards_stay_refused(which):
    b200, m, fc, att, labels, masks, gts = _newfc()
    lw = b200.B200LossWrapper(m, _wrapper_opt(bleu_reward_weight=0.5, **{which: 0.1}))
    lw._scorer = lambda: None
    with pytest.raises(NotImplementedError, match='self-CIDEr'):
        lw(fc, att, labels, masks, None, gts, torch.arange(2), False, True, False)
    crit = b200.loss_wrapper.StructureLosses(_wrapper_opt(train_sample_n=1, **{which: 0.1}))
    with pytest.raises(NotImplementedError, match='self-CIDEr'):
        crit(torch.zeros(2, 5, 31), torch.zeros(2, 5, dtype=torch.long), gts)
