"""Att2in2 without a GPU: the restatement in att2in2_oracle against the live-reference goldens, the Python mirror's parameter names, the
C-ABI weight table layout, and the refusals that must happen before any device work."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from helpers import co, family_opt
import att2in2_oracle as ao
import dbs_oracle

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def small_setup():
    g = np.load(os.path.join(GOLD, 'att2in2_small.npz'))
    meta = json.loads(str(g['meta']))
    V, E, H, A, F_fc, F_att, T = (int(x) for x in g['cfg'])
    W = co.make_weights('att2in2', V, E, H, A, F_fc, F_att, seed=meta['seed'], logit_scale=meta['logit_scale'])
    fc, att = co.make_inputs(meta['B'], meta['R'], F_fc, F_att, seed=meta['seed'])
    masks = torch.ones(meta['B'], meta['R'])
    masks[1, 5:] = 0
    masks[3, 3:] = 0
    return g, meta, W, fc, att, masks, T


def test_restatement_decode_goldens():
    g, meta, W, fc, att, masks, T = small_setup()
    fam = ao.Att2in2Family(W, T)
    for tag, mk in (('', None), ('masked_', masks)):
        seq, lp = co.sample(fam, fc, att, mk)
        assert np.array_equal(seq.numpy(), g[tag + 'greedy_seq'])
        np.testing.assert_allclose(lp.numpy(), g[tag + 'greedy_lp'], rtol=0, atol=1e-5)
    sseq = torch.from_numpy(g['sample_seq'])
    _, lp = co.sample(fam, fc, att, sample_n=3, forced_tokens=sseq)
    np.testing.assert_allclose(lp.numpy(), g['sample_lp'], rtol=0, atol=1e-5)
    labels = torch.from_numpy(g['tf_labels'])
    lp = co.forward_teacher(fam, fc, att, labels[:, :-1].reshape(fc.shape[0], 2, -1))
    np.testing.assert_allclose(lp.numpy(), g['tf_lp'], rtol=0, atol=1e-5)


@pytest.mark.parametrize('case', ['beam_wu', 'beam_constraint', 'beam_masked', 'dbs'])
def test_restatement_beam_goldens(case):
    g, meta, W, fc, att, masks, T = small_setup()
    fam = ao.Att2in2Family(W, T)
    mk = masks if case == 'beam_masked' else None
    if case == 'dbs':
        seq, lp, done = dbs_oracle.diverse_sample_beam(fam, fc, att, beam_size=6, group_size=3, diversity_lambda=0.5)
        beam = 6
    else:
        beam = 4
        if case == 'beam_constraint':      # co.beam_search has no decoding_constraint: the diverse restatement with one group does
            seq, lp, done = dbs_oracle.diverse_sample_beam(fam, fc, att, mk, beam_size=4, group_size=1, decoding_constraint=True)
        else:
            seq, lp, done = co.sample_beam(fam, fc, att, mk, beam_size=4, length_penalty='wu_0.5' if case == 'beam_wu' else '')
    assert np.array_equal(seq.numpy(), g[case + '_seq'])
    dseq, dlen, dp = dbs_oracle.beams_to_arrays(done, beam, T)
    assert np.array_equal(dseq, g[case + '_done_seq']) and np.array_equal(dlen, g[case + '_done_len'])
    assert np.abs(dp - g[case + '_done_p']).max() < 1e-4
    for j, rec in enumerate(done[0]):
        L = rec['logps'].shape[0]
        np.testing.assert_allclose(rec['logps'].numpy(), g[case + '_logps0'][j, :L], rtol=0, atol=1e-5)


def _oracle_train_grads(W, fc, att, masks, T, kind, g):
    Wg = {k: v.clone().requires_grad_(True) for k, v in W.items()}
    fam = ao.Att2in2Family(Wg, T)
    B = fc.shape[0]
    if kind == 'xe':
        labels, lmasks = torch.from_numpy(g['xe_labels']), torch.from_numpy(g['xe_masks'])
        lp = co.forward_teacher(fam, fc, att, labels[:, :-1].reshape(B, 3, -1), masks)
        loss = co.language_model_criterion(lp, labels[:, 1:], lmasks[:, 1:])
    else:
        seq = torch.from_numpy(g['rl_seq'])
        _, lp = co.sample(fam, fc, att, masks, sample_method='sample', sample_n=3, forced_tokens=seq)
        loss = co.reward_criterion(lp, seq, torch.from_numpy(g['rl_reward']))
    loss.backward()
    return float(loss), {k: v.grad for k, v in Wg.items()}


@pytest.mark.parametrize('kind', ['xe', 'rl'])
def test_restatement_training_goldens(kind):
    """Autograd through the restatement reproduces the reference's loss.backward() for every one of the 17 parameters."""
    g, meta, W, fc, att, masks, T = small_setup()
    loss, grads = _oracle_train_grads(W, fc, att, masks, T, kind, g)
    assert abs(loss - float(g[kind + '_loss'])) < 1e-5
    assert sorted(grads) == sorted(meta['params']) and len(grads) == 17
    for k, v in grads.items():
        ref = g['%s_grad_%s' % (kind, k)]
        assert np.abs(v.numpy() - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max()), k


def test_restatement_recipe_beam_golden():
    """Tie-aware: ids must agree on every image whose smallest candidate gap is clear of float noise."""
    g = np.load(os.path.join(GOLD, 'att2in2_b32.npz'))
    V, E, H, A, F_fc, F_att, T = (int(x) for x in g['cfg'])
    B, R, beam, seed = (int(x) for x in g['meta'])
    assert (V, E, H, A, T, beam) == (9487, 512, 512, 512, 20, 5)
    # the full-size restatement takes a while on the CPU: check the first images only
    nb = 4
    W = co.make_weights('att2in2', V, E, H, A, F_fc, F_att, seed=seed, logit_scale=12.0)
    fc, att = co.make_inputs(B, R, F_fc, F_att, seed=seed)
    _, _, done = co.sample_beam(ao.Att2in2Family(W, T), fc[:nb], att[:nb], beam_size=beam)
    dseq, _, dp = dbs_oracle.beams_to_arrays(done, beam, T)
    clear = g['image_margin'][:nb] > 1e-4
    assert clear.any()
    assert np.array_equal(dseq[clear], g['done_seq'][:nb][clear].astype(np.int64))
    assert np.abs(dp[:, 0] - g['done_p'][:nb, 0]).max() < 1e-3


def test_state_dict_keys_match_reference():
    import imagecaptioning.pytorch_b200 as b200
    ref = json.load(open(os.path.join(GOLD, 'att2in2_state_dict_keys.json')))
    c = ref['cfg']
    m = b200.setup(family_opt('att2in2', c['V'], c['E'], c['H'], c['A'], c['F_fc'], c['F_att'], c['T']))
    assert {k: list(v.shape) for k, v in m.state_dict().items()} == ref['keys']
    W = co.make_weights('att2in2', c['V'], c['E'], c['H'], c['A'], c['F_fc'], c['F_att'], seed=1)
    assert {k: list(v.shape) for k, v in W.items()} == ref['keys']
    assert set(m._weight_table()) == set(b200._lib.ATT2IN2_GRAD_FIELDS)


@pytest.mark.skipif(torch.cuda.is_available(), reason='checks the behaviour of a box without a GPU')
def test_cpu_tensors_raise():
    import imagecaptioning.pytorch_b200 as b200
    m = b200.setup(family_opt('att2in2', 30, 16, 16, 8, 16, 16, 5))
    with pytest.raises(RuntimeError, match='CUDA'):
        m(torch.zeros(2, 16), torch.zeros(2, 3, 16), None, opt={'beam_size': 1}, mode='sample')
    with pytest.raises(RuntimeError, match='CUDA'):
        m(torch.zeros(2, 16), torch.zeros(2, 3, 16), None, opt={'beam_size': 4, 'group_size': 2, 'sample_n': 1}, mode='sample')


def test_refusals_before_device_work():
    import argparse
    import imagecaptioning.pytorch_b200 as b200
    m = b200.setup(family_opt('att2in2', 30, 16, 16, 8, 16, 16, 5))
    fc, att = torch.zeros(2, 16), torch.zeros(2, 3, 16)
    for bad in ({'group_size': 2, 'beam_size': 1}, {'output_logsoftmax': 0}):
        with pytest.raises(NotImplementedError):
            m(fc, att, None, opt=bad, mode='sample')
    opt = argparse.Namespace(structure_loss_type="seqnll", structure_loss_weight=1.0, train_sample_n=2, cider_reward_weight=1.0, bleu_reward_weight=0.0, sc_sample_method='greedy',
                             sc_beam_size=1, train_sample_method='sample', train_beam_size=1, structure_after=-1, label_smoothing=0.0)
    lw = b200.B200LossWrapper(m, opt)
    labels, masks = torch.zeros(2, 7, dtype=torch.long), torch.ones(2, 7)
    with pytest.raises(NotImplementedError):
        lw(fc, att, labels, masks, None, [np.zeros((1, 5), np.int64)] * 2, torch.arange(2), False, True, False)
    for name in ('att2in', 'att2all2', 'adaatt'):
        with pytest.raises(NotImplementedError):
            b200.setup(family_opt(name, 30, 16, 16, 8, 16, 16, 5))


def test_weights_struct_grew_by_two_pointers():
    """a2c_w / a2c_b are appended: the existing fields keep their offsets (the ABI version stays 1)."""
    import imagecaptioning.pytorch_b200 as b200
    W = b200._lib.Weights
    assert ctypes.sizeof(W) == 27 * 8 and ctypes.sizeof(W) - 25 * 8 == 16
    for i, f in enumerate(b200._lib.WEIGHT_FIELDS[:25]):
        assert getattr(W, f).offset == 8 * i
    assert W.a2c_w.offset == 200 and W.a2c_b.offset == 208
