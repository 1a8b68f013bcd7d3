"""NewFC training without a GPU: the restatement in newfc_oracle against the live-reference training goldens (tests/make_newfc_golden.py),
the C-ABI gradient table layout, and the loss wrapper's dispatch of NewFC's XE, sc and struc branches to the fused steps."""
import argparse
import json
import os
import re

import numpy as np
import pytest
import torch

from helpers import REPO, co, family_opt
import newfc_oracle as no

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def df_of(g):
    """The document-frequency dict stored with a golden (keys padded with -1)."""
    return {tuple(int(t) for t in k if t >= 0): float(v) for k, v in zip(g['df_keys'], g['df_vals'])}, float(g['ref_len'])


def fingerprint_err(grad, sub, step, stats):
    """Largest deviation of a gradient from its stored _subsample fingerprint (sub-grid and sum / abs-sum / norm / max), relative to the
    tensor's largest entry."""
    a = grad.detach().numpy()
    mine = a.copy() if a.size == sub.size and a.shape == sub.shape else (a[::step[0]] if a.ndim == 1 else a[::step[0], ::step[1]])
    scale = float(stats[3])
    err = float(np.abs(mine - sub).max()) / scale
    st = np.array([a.sum(dtype=np.float64), np.abs(a).sum(dtype=np.float64), np.sqrt((a.astype(np.float64) ** 2).sum()), np.abs(a).max()])
    err = max(err, abs(st[3] - stats[3]) / scale, abs(st[2] - stats[2]) / max(stats[2], 1e-30))
    err = max(err, abs(st[0] - stats[0]) / (stats[1] + 1e-30))
    return err


def small_setup():
    g = np.load(os.path.join(GOLD, 'newfc_train_small.npz'))
    meta = json.loads(str(g['meta']))
    V, E, H, A, F_fc, F_att, T = (int(x) for x in g['cfg'])
    W = co.make_weights('newfc', V, E, H, A, F_fc, F_att, seed=meta['seed'], logit_scale=meta['logit_scale'])
    fc, _ = co.make_inputs(meta['B'], 1, F_fc, F_att, seed=meta['seed'])
    return g, meta, W, fc, fc.new_zeros(meta['B'], 0, 0), T


def small_oracle(W, fc, att, T, kind, g):
    Wg = {k: v.clone().requires_grad_(True) for k, v in W.items()}
    fam = no.NewFCFamily(Wg, T)
    B = fc.shape[0]
    if kind in ('xe', 'ls'):
        labels, lmasks = torch.from_numpy(g['xe_labels']), torch.from_numpy(g['xe_masks'])
        lp = co.forward_teacher(fam, fc, att, labels[:, :-1].reshape(B, 3, -1))
        if kind == 'xe':
            loss = co.language_model_criterion(lp, labels[:, 1:], lmasks[:, 1:])
        else:
            loss = co.label_smoothing_loss(lp, labels[:, 1:], lmasks[:, 1:], 0.2)
    else:
        seq = torch.from_numpy(g['rl_seq'])
        _, lp = co.sample(fam, fc, att, sample_method='sample', sample_n=3, forced_tokens=seq)
        loss = co.reward_criterion(lp, seq, torch.from_numpy(g['rl_reward']))
    loss.backward()
    return float(loss), {k: v.grad for k, v in Wg.items()}, lp.detach()


@pytest.mark.parametrize('kind', ['xe', 'ls', 'rl'])
def test_restatement_small_golden(kind):
    """Autograd through the restatement reproduces the reference's loss.backward() for every one of the 9 parameters (att_feats [B, 0, 0])."""
    g, meta, W, fc, att, T = small_setup()
    loss, grads, lp = small_oracle(W, fc, att, T, kind, g)
    assert abs(loss - float(g[kind + '_loss'])) < 1e-5
    assert sorted(grads) == sorted(meta['params']) and len(grads) == 9
    for k, v in grads.items():
        ref = g['%s_grad_%s' % (kind, k)]
        assert np.abs(ref).max() > 0, k
        assert np.abs(v.numpy() - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max()), k
    if kind == 'rl':
        np.testing.assert_allclose(lp.numpy(), g['rl_lp'], rtol=0, atol=1e-5)


def full_setup():
    g = np.load(os.path.join(GOLD, 'newfc_scst_full.npz'))
    V, E, H, A, F_fc, F_att, T = (int(x) for x in g['cfg'])
    B, n, seed = (int(x) for x in g['meta'])
    W = co.make_weights('newfc', V, E, H, A, F_fc, F_att, seed=seed, logit_scale=float(g['logit_scale']))
    fc, _ = co.make_inputs(B, 1, F_fc, F_att, seed=seed)
    gts = [r.astype(np.int64) for r in g['gts']]
    return g, W, fc, fc.new_zeros(B, 0, 0), gts, B, n, T


def full_oracle(g, W, fc, att, gts, B, n, T, branch):
    """(loss, per-sample reward / score, gradients, greedy caption) of the restatement replaying the reference's samples."""
    from oracle import ciderd_oracle as cdo
    df, ref_len = df_of(g)
    seq = torch.from_numpy(g[branch + '_sample_seq'].astype(np.int64))
    greedy = None
    if branch == 'sc':
        greedy, _ = co.sample(no.NewFCFamily(W, T), fc, att)
        reward, _ = cdo.self_critical_reward(greedy.numpy(), gts, seq.numpy(), df, ref_len)
        reward = torch.from_numpy(reward).float()
        per = reward[:, 0].double().numpy()
    else:
        scores = torch.from_numpy(cdo.get_scores(gts, seq.numpy(), df, ref_len))
        per = scores.numpy()
    Wg = {k: v.clone().requires_grad_(True) for k, v in W.items()}
    _, lp = co.sample(no.NewFCFamily(Wg, T), fc, att, sample_method='sample', sample_n=n, forced_tokens=seq)
    loss = co.reward_criterion(lp, seq, reward) if branch == 'sc' else co.new_self_critical_loss(lp, seq, scores, n)
    loss.backward()
    return float(loss), per, {k: v.grad for k, v in Wg.items()}, greedy


@pytest.mark.parametrize('branch', ['sc', 'nsc'])
def test_restatement_recipe_golden(branch):
    """fc_rl / fc_nsc recipe size (10 images x 5 samples, E = H = 512, V = 9487): the reference's LossWrapper step and backward() are
    reproduced on loss, rewards and every gradient fingerprint."""
    g, W, fc, att, gts, B, n, T = full_setup()
    assert (B, n, T) == (10, 5, 20) and int(g['cfg'][1]) == 512 and int(g['cfg'][0]) == 9487
    loss, per, grads, greedy = full_oracle(g, W, fc, att, gts, B, n, T, branch)
    assert abs(loss - float(g[branch + '_loss'])) < 1e-4 * max(1.0, abs(float(g[branch + '_loss'])))
    if branch == 'sc':
        assert np.array_equal(greedy.numpy(), g['sc_greedy_seq'].astype(np.int64))
        assert np.abs(per - g['sc_reward']).max() < 1e-4
    else:
        assert np.abs(per - g['nsc_scores']).max() < 1e-4
    names = [str(k) for k in g['names']]
    assert sorted(names) == sorted(grads) and len(names) == 9
    for k in names:
        err = fingerprint_err(grads[k], g['%s_g_%s' % (branch, k)], g['%s_s_%s' % (branch, k)], g['%s_t_%s' % (branch, k)])
        assert err < 5e-5, (k, err)


def test_grads_struct_matches_header():
    """NewfcGrads has the fields of capb200_newfc_grads in include/capb200.h, in order."""
    import imagecaptioning.pytorch_b200 as b200
    hdr = open(os.path.join(REPO, 'include', 'capb200.h')).read()
    body = re.search(r'typedef struct \{([^}]*)\} capb200_newfc_grads;', hdr).group(1)
    fields = re.findall(r'\*\s*(\w+)', body)
    assert fields == b200._lib.NEWFC_GRAD_FIELDS == [f for f, _ in b200._lib.NewfcGrads._fields_]
    assert fields == ['embed', 'fc_embed_w', 'fc_embed_b', 'logit_w', 'logit_b', 'i2h_w', 'i2h_b', 'h2h_w', 'h2h_b']
    m = b200.setup(family_opt('newfc', 30, 16, 16, 8, 16, 16, 5))
    assert set(m._weight_table()) == set(fields)
    assert not isinstance(m, b200.B200UpDownModel)


def _wrapper_opt(**kw):
    opt = dict(sc_sample_method='greedy', sc_beam_size=1, train_sample_method='sample', train_beam_size=1, train_sample_n=5, cider_reward_weight=1,
               bleu_reward_weight=0, structure_loss_type='new_self_critical', structure_loss_weight=1.0, label_smoothing=0.0, use_ppo=0)
    opt.update(kw)
    return argparse.Namespace(**opt)


@pytest.mark.skipif(torch.cuda.is_available(), reason='checks the behaviour of a box without a GPU')
@pytest.mark.parametrize('branch', ['xe', 'sc', 'struc'])
def test_loss_wrapper_dispatches_to_fused_steps(branch):
    """fc.yml (XE), fc_rl.yml (sc) and fc_nsc.yml (struc, new_self_critical) option sets reach NewFC's fused steps: no NotImplementedError,
    the call stops at the engine's refusal of CPU tensors.  att_feats is what the reference loader hands NewFC: [B, 0, 0]."""
    import imagecaptioning.pytorch_b200 as b200
    m = b200.setup(family_opt('newfc', 30, 16, 16, 8, 16, 16, 5)).train()
    B = 2
    fc, att = torch.zeros(B, 16), torch.zeros(B, 0, 0)
    labels, masks = torch.zeros(B, 5, 7, dtype=torch.long), torch.ones(B, 5, 7)
    labels[:, :, 1] = 3
    lw = b200.B200LossWrapper(m, _wrapper_opt())
    lw._scorer = lambda: None           # the CIDEr-D table lives on a GPU; the step refuses the CPU tensors before it would read it
    gts = [np.ones((1, 5), np.int64)] * B
    with pytest.raises(RuntimeError, match='CUDA'):
        lw(fc, att, labels, masks, None, gts, torch.arange(B), branch == 'sc', branch == 'struc', False)


def test_refusals_stay():
    """Diverse beam search, output_logsoftmax=0 and structure losses other than new_self_critical stay refused for NewFC."""
    import imagecaptioning.pytorch_b200 as b200
    m = b200.setup(family_opt('newfc', 30, 16, 16, 8, 16, 16, 5))
    fc, att = torch.zeros(2, 16), torch.zeros(2, 0, 0)
    for bad in ({'beam_size': 4, 'group_size': 2, 'sample_n': 1}, {'output_logsoftmax': 0}):
        with pytest.raises(NotImplementedError):
            m(fc, att, None, opt=bad, mode='sample')
    lw = b200.B200LossWrapper(m.train(), _wrapper_opt(structure_loss_type='seqnll'))
    labels, masks = torch.zeros(2, 7, dtype=torch.long), torch.ones(2, 7)
    with pytest.raises(NotImplementedError):
        lw(fc, att, labels, masks, None, [np.zeros((1, 5), np.int64)] * 2, torch.arange(2), False, True, False)
