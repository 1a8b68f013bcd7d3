"""PPO (use_ppo) without a GPU: the repo's PPO oracle against the live reference's PPOLoss (tests/golden/ppo_small.npz, from
tests/make_ppo_golden.py), the UpDown oracle's teacher-forced old-policy pass against the reference's, and what B200LossWrapper does
before any device work: the old policy it builds (or does not build) and the configurations it refuses."""
import argparse
import os

import numpy as np
import pytest
import torch

from helpers import REPO, co, family_opt
from ppo_oracle import old_policy_input, ppo_loss

GOLD = os.path.join(REPO, 'tests', 'golden', 'ppo_small.npz')
CFG = dict(V=30, E=16, H=16, A=8, F_fc=12, F_att=12, T=7)


def _gold():
    g = np.load(GOLD)
    W = {k[2:]: torch.from_numpy(g[k]) for k in g.files if k.startswith('w:')}
    return g, W


@pytest.mark.parametrize('reduction', ['mean', 'none'])
def test_oracle_matches_reference(reduction):
    g, _ = _gold()
    B, n, _ = (int(x) for x in g['dims'])
    eps, kl_coef = (float(x) for x in g['hyper'])
    lp = torch.from_numpy(g['lp']).double().requires_grad_(True)
    out = ppo_loss(lp, torch.from_numpy(g['lo']).double(), torch.from_numpy(g['seq']), torch.from_numpy(g['scores']), n, eps, kl_coef, reduction)
    (out['loss'] if reduction == 'mean' else out['loss'].sum()).backward()
    for k in ('loss', 'pg_loss', 'kl_loss', 'clipfrac', 'reward'):
        assert np.abs(out[k].detach().numpy() - g['%s_%s' % (reduction, k)]).max() < 2e-6, k
    want = g['%s_dlp' % reduction]
    assert np.abs(lp.grad.numpy() - want).max() < 2e-6 * max(1.0, np.abs(want).max())
    assert 0.0 < float(g['mean_clipfrac']) < 1.0          # both sides of the clip range are exercised


def test_old_policy_pass_matches_reference():
    """The reference's old model (copy.deepcopy + load_state_dict of the saved weights, eval mode) against co.forward_teacher over
    [0, seq[:, :-1]] with the same weights."""
    g, W = _gold()
    seq = torch.from_numpy(g['seq'])
    B, n, _ = (int(x) for x in g['dims'])
    lo = co.forward_teacher(co.Family('updown', W, CFG['T']), torch.from_numpy(g['fc']), torch.from_numpy(g['att']),
                            old_policy_input(seq).reshape(B, n, -1))
    m = torch.cat([torch.ones(seq.shape[0], 1, dtype=torch.bool), seq[:, :-1] > 0], 1)
    assert float((lo - torch.from_numpy(g['lo']))[m].abs().max()) < 1e-5


def _opt(**kw):
    base = dict(use_ppo=1, ppo_old_model_path=None, ppo_cliprange=0.2, ppo_kl_coef=0.02, train_sample_n=3, train_sample_method='sample',
                train_beam_size=1, sc_sample_method='greedy', sc_beam_size=1, structure_loss_type='new_self_critical', structure_loss_weight=1.0,
                label_smoothing=0.0, struc_use_logsoftmax=1, entropy_reward_weight=0, self_cider_reward_weight=0)
    base.update(kw)
    return argparse.Namespace(**base)


def _model(seed=5):
    import imagecaptioning.pytorch_b200 as b200
    dims = tuple(CFG[k] for k in ('V', 'E', 'H', 'A', 'F_fc', 'F_att', 'T'))
    m = b200.setup(family_opt('updown', *dims))
    m.load_state_dict(co.make_weights('updown', *dims[:6], seed=seed, logit_scale=4.0), strict=True)
    return m


def _saved(tmp_path, lightning):
    old = _model(seed=6).state_dict()
    path = str(tmp_path / ('old.ckpt' if lightning else 'old.pth'))
    if lightning:
        sd = dict(old, _vocab={'1': 'w1'}, _opt=argparse.Namespace(caption_model='updown'))
        torch.save({'pytorch-lightning_version': '1.5.0', 'state_dict': sd, 'epoch': 3}, path)
    else:
        torch.save(old, path)
    return path, old


@pytest.mark.parametrize('lightning', [False, True])
def test_wrapper_builds_the_frozen_old_policy(tmp_path, lightning):
    import imagecaptioning.pytorch_b200 as b200
    path, want = _saved(tmp_path, lightning)
    model = _model()
    before = {k: v.clone() for k, v in model.state_dict().items()}
    lw = b200.B200LossWrapper(model, _opt(ppo_old_model_path=path))
    old = lw.old_model
    assert type(old) is type(model) and old is not model and not old.training
    assert all(not p.requires_grad for p in old.parameters())
    for k, v in old.state_dict().items():
        assert torch.equal(v, want[k]), k
    for k, v in model.state_dict().items():
        assert torch.equal(v, before[k]), k
    assert any(not torch.equal(before[k], want[k]) for k in want)


def test_wrapper_without_ppo_builds_no_old_model():
    import imagecaptioning.pytorch_b200 as b200
    assert b200.B200LossWrapper(_model(), _opt(use_ppo=0)).old_model is None
    assert b200.B200LossWrapper(_model(), argparse.Namespace(label_smoothing=0.0)).old_model is None


def test_wrapper_needs_the_old_model_path():
    import imagecaptioning.pytorch_b200 as b200
    with pytest.raises(AssertionError, match='old model path'):
        b200.B200LossWrapper(_model(), _opt())


@pytest.mark.parametrize('kw', [dict(structure_loss_type='margin', struc_use_logsoftmax=0), dict(train_beam_size=2, train_sample_method='greedy'),
                                dict(entropy_reward_weight=0.5), dict(self_cider_reward_weight=0.5), dict(train_sample_method='beam_search')],
                         ids=['logits', 'beam', 'entropy', 'self_cider', 'beam_method'])
def test_wrapper_refuses_before_device_work(tmp_path, kw):
    """PPO on logits, beam-search samples and the entropy / self-CIDEr reward terms raise NotImplementedError on CPU tensors, i.e. before the
    engine is touched."""
    import imagecaptioning.pytorch_b200 as b200
    path, _ = _saved(tmp_path, False)
    lw = b200.B200LossWrapper(_model(), _opt(ppo_old_model_path=path, **kw))
    B, T = 2, CFG['T']
    fc, att = co.make_inputs(B, 4, CFG['F_fc'], CFG['F_att'], seed=1)
    labels = torch.zeros(B, 3, T + 2, dtype=torch.long)
    gts = [np.ones((1, T), np.int64)] * B
    with pytest.raises(NotImplementedError):
        lw(fc, att, labels, torch.ones(B, 3, T + 2), None, gts, torch.arange(B), False, True, False)


def test_ppo_step_refuses_another_old_model():
    import imagecaptioning.pytorch_b200 as b200
    model = _model()
    dims = (CFG['V'], CFG['E'], CFG['H'], CFG['A'], CFG['F_fc'], CFG['F_att'], CFG['T'])
    other = b200.setup(family_opt('att2in2', *dims))
    wider = b200.setup(family_opt('updown', *dims[:2], CFG['H'] * 2, *dims[3:]))
    fc, att = co.make_inputs(2, 4, CFG['F_fc'], CFG['F_att'], seed=1)
    for old in (model, other, wider):
        with pytest.raises(ValueError, match='old model'):
            model.ppo_step(old, fc, att, [np.ones((1, 3), np.int64)] * 2, None, 3)
    ens = b200.B200AttEnsemble([_model(), _model(seed=6)])
    with pytest.raises(NotImplementedError):
        ens.ppo_step(ens, fc, att, [np.ones((1, 3), np.int64)] * 2, None, 3)
