"""PPO (use_ppo) on the H100: every family's fused ppo_step against autograd through the family's oracle -- the new policy's sampled pass,
the old policy's teacher-forced pass over [0, seq[:, :-1]], then the PPO oracle (tests/ppo_oracle.py, held to the live reference by
test_ppo_cpu.py) -- and B200LossWrapper with use_ppo over saved and Lightning-format old-policy checkpoints.  The samples are the oracle's
own seeded draw, replayed as forced tokens."""
import argparse

import numpy as np
import pytest
import torch

from helpers import LOGP_TOL, co, dropout_masks, family_opt
import att2in2_oracle as ao
import bleu_oracle as bo
import newfc_oracle as no
from ppo_oracle import old_policy_input, ppo_loss, token_mask

pytestmark = pytest.mark.gpu

RNN_CFG = dict(V=40, E=32, H=48, A=24, F_fc=32, F_att=40, T=9)
AOA_CFG = dict(V=40, E=32, H=64, A=0, F_fc=32, F_att=40, T=7)
TFM_CFG = dict(V=40, E=32, H=64, A=2, F_fc=32, F_att=40, T=7)
BIG_CFG = dict(RNN_CFG, V=52000)          # V + 1 > 51 199: the thread-block-cluster vocabulary step
HEADS = 4
FAMILIES = ['updown', 'att2in2', 'newfc', 'aoa', 'transformer']
GRAD_REL = 5e-4
EPS, KL_COEF = 0.2, 0.02
R_FEATS = 9
# the old policy's weights are the new ones plus this much noise (relative to each tensor's spread): chosen so that some policy ratios of each
# case leave the clip range and none lies within 1e-3 of its edges on the oracle (test_ppo_step_perturbed_old_policy asserts a 1e-4 margin)
PERTURB = {'updown': 0.35, 'att2in2': 0.25, 'newfc': 0.15, 'aoa': 0.15, 'transformer': 0.02}


def _cfg(name, big=False):
    return BIG_CFG if big else {'aoa': AOA_CFG, 'transformer': TFM_CFG}.get(name, RNN_CFG)


def _oracle(name, cfg):
    if name == 'att2in2':
        return lambda w: ao.Att2in2Family(w, cfg['T'])
    if name == 'newfc':
        return lambda w: no.NewFCFamily(w, cfg['T'])
    return lambda w: co.Family(name, w, cfg['T'], heads=HEADS)


def _weights(name, cfg, perturb=0.0, seed=21):
    W = co.make_weights(name, *(cfg[k] for k in ('V', 'E', 'H', 'A', 'F_fc', 'F_att')), seed=seed, logit_scale=5.0)
    if perturb:
        g = torch.Generator().manual_seed(seed + 1)
        W = {k: v if k.endswith('.pe') else v + perturb * (v.std() if v.numel() > 1 else 1.0) * torch.randn(v.shape, generator=g)
             for k, v in W.items()}
    return W


def _case(name, B=3, n=4, perturb=0.0, region_mask=False, big=False, seed=4):
    """(cfg, new weights, old weights, fc, att, region mask or None, samples [B*n, T]): the oracle's own multinomial draw of the new policy."""
    cfg = _cfg(name, big)
    W, W_old = _weights(name, cfg), _weights(name, cfg, perturb)
    fc, att = co.make_inputs(B, R_FEATS, cfg['F_fc'], cfg['F_att'], seed=seed)
    if name == 'newfc':
        att = fc.new_zeros(B, 0, 0)
    masks = None
    if region_mask:
        masks = torch.ones(B, R_FEATS)
        for i in range(B):
            masks[i, R_FEATS - 2 * i:] = 0
    torch.manual_seed(seed)
    with torch.no_grad():
        seq, _ = co.sample(_oracle(name, cfg)(W), fc, att, masks, sample_method='sample', sample_n=n)
    return cfg, W, W_old, fc, att, masks, seq


def _engine(name, cfg, W):
    import imagecaptioning.pytorch_b200 as b200
    model = b200.setup(family_opt(name, *(cfg[k] for k in ('V', 'E', 'H', 'A', 'F_fc', 'F_att', 'T')), heads=HEADS), numeric_mode='tc_f16x3')
    model.load_state_dict(W, strict=True)
    return model.cuda()


def _scorer(cfg):
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    df, ref_len = cdo.build_document_frequency(cdo.make_refs(200, cfg['V'], seed=4))
    return df, ref_len, b200.rewards.CiderDTable(df, ref_len)


def _rates(name, p=0.0):
    kw = dict(drop_prob=p)
    if name == 'aoa':
        kw.update(drop_attn=0.0, drop_aoa=0.0, drop_sublayer=0.0)
    if name == 'transformer':
        kw.update(dropout=0.0)
    return kw


def _ratios(lp, lo, seq):
    idx = seq.unsqueeze(2)
    r = torch.exp(lp.gather(2, idx) - lo.gather(2, idx)).squeeze(2)
    return r[token_mask(seq) > 0]


def _check_grads(model, grads, Wg, rel=GRAD_REL):
    name_of = {id(p): k for k, p in model.state_dict(keep_vars=True).items()}
    ograds = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in Wg.items() if v.requires_grad}
    largest = max(float(v.abs().max()) for v in ograds.values())
    for p, g in grads.items():
        key = name_of[id(p)]
        ref = ograds[key]
        err = float((g.cpu() - ref).abs().max())
        assert err <= rel * float(ref.abs().max()) + 1e-7 * largest, (key, err)
    assert sum(float(v.abs().max()) > 1e-6 for v in ograds.values()) >= len(grads) // 2


def _run(name, B=3, n=4, perturb=0.0, region_mask=False, big=False, keep=0, weights=None, drop_prob=0.0, seed=4):
    """One ppo_step against the oracle; returns (result, oracle ratios at the live positions)."""
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    cfg, W, W_old, fc, att, masks, seq = _case(name, B, n, perturb, region_mask, big, seed)
    model, old = _engine(name, cfg, W).train(), _engine(name, cfg, W_old).eval()
    gts = cdo.make_refs(B, cfg['V'], seed=2)
    if big:     # random references share no n-gram with the samples of a 52 000-word vocabulary: each image's first sample becomes one
        for i in range(B):
            gts[i][0, :] = 0
            gts[i][0, :cfg['T']] = seq[i * n].numpy()
    df, ref_len, table = _scorer(cfg)
    step_seed = 4321
    res = model.ppo_step(old, fc.cuda(), att.cuda(), gts, table, n, cliprange=EPS, kl_coef=KL_COEF, seed=step_seed, forced_tokens=seq.cuda(),
                         att_masks=None if masks is None else masks.cuda(), keep_rows=keep, reward_weights=weights, **_rates(name, drop_prob))
    torch.cuda.synchronize()
    assert torch.equal(res['sample_seq'].cpu(), seq)
    Wg = {k: (v.clone() if k.endswith('.pe') else v.clone().requires_grad_(True)) for k, v in W.items()}
    fam = _oracle(name, cfg)(Wg)
    if drop_prob > 0:       # the step's dropout masks, replayed (UpDown's sites)
        fam.drop = dropout_masks(b200, step_seed, drop_prob, B, R_FEATS, B * n, cfg['T'], cfg['E'], cfg['H'])
    _, lp = co.sample(fam, fc, att, masks, sample_method='sample', sample_n=n, forced_tokens=seq)
    with torch.no_grad():
        lo = co.forward_teacher(_oracle(name, cfg)(W_old), fc, att, old_policy_input(seq).reshape(B, n, -1), masks)
    scores = torch.from_numpy(bo.get_scores(gts, seq.numpy(), weights or (1.0, 0.0), df, ref_len))
    out = ppo_loss(lp, lo, seq, scores, n, EPS, KL_COEF, 'none' if keep else 'mean')
    loss = out['loss'].sort().values[:keep].mean() if keep else out['loss']
    loss.backward()
    assert float((res['sample_logprobs'].cpu() - lp.detach()).abs().max()) < LOGP_TOL
    assert float((res['scores'].cpu() - scores.float().view(B, n)).abs().max()) < 1e-5
    assert abs(float(res['loss']) - float(loss.detach())) < LOGP_TOL
    for k in ('pg_loss', 'kl_loss', 'clipfrac'):
        assert abs(float(res[k]) - float(out[k].detach())) < LOGP_TOL, k
    if keep:
        assert float((res['row_loss'].cpu() - out['loss'].detach()).abs().max()) < LOGP_TOL
    sc = scores.view(B, n)
    assert float((sc - sc.mean(1, keepdim=True)).abs().max()) > 1e-3        # not vacuous: the advantage is not zero
    _check_grads(model, res['grads'], Wg)
    return res, _ratios(lp.detach(), lo, seq)


@pytest.mark.parametrize('family', FAMILIES)
def test_ppo_step_old_equals_new(family):
    """The old policy holds the new one's weights: without dropout every ratio is 1 up to rounding, the loss is the leave-one-out policy
    gradient and kl_loss ~ 0."""
    res, ratio = _run(family)
    assert float((ratio - 1).abs().max()) < 1e-4
    assert float(res['clipfrac']) == 0.0 and abs(float(res['kl_loss'])) < 1e-4


def test_ppo_step_dropout_moves_the_ratio():
    """Old = new weights, dropout 0.5 in the new policy's sampled pass only (the old policy runs in eval mode): the ratios leave 1."""
    _, ratio = _run('updown', drop_prob=0.5)
    assert float((ratio - 1).abs().max()) > 1e-2


@pytest.mark.parametrize('family', FAMILIES)
def test_ppo_step_perturbed_old_policy(family):
    res, ratio = _run(family, perturb=PERTURB[family])
    assert 0.0 < float(res['clipfrac']) < 1.0
    assert float(torch.minimum((ratio - (1 - EPS)).abs(), (ratio - (1 + EPS)).abs()).min()) > 1e-4


@pytest.mark.parametrize('family', FAMILIES)
def test_ppo_step_drop_worst(family):
    _run(family, perturb=PERTURB[family], keep=7)


@pytest.mark.parametrize('family', ['aoa', 'transformer', 'updown'])
def test_ppo_step_region_mask(family):
    _run(family, perturb=PERTURB[family], region_mask=True, weights=(0.7, 0.3))


def test_ppo_step_large_vocabulary():
    res, _ = _run('updown', B=2, n=2, perturb=PERTURB['updown'], big=True)
    assert res['sample_logprobs'].shape[2] > 51199


def _lw_opt(n, path, w):
    return argparse.Namespace(use_ppo=1, ppo_old_model_path=path, ppo_cliprange=EPS, ppo_kl_coef=KL_COEF, train_sample_n=n,
                              train_sample_method='sample', train_beam_size=1, sc_sample_method='greedy', sc_beam_size=1,
                              structure_loss_type='new_self_critical', structure_loss_weight=w, label_smoothing=0.0)


@pytest.mark.parametrize('lightning', [False, True])
@pytest.mark.parametrize('w', [1.0, 0.5])
def test_loss_wrapper_ppo(tmp_path, lightning, w):
    """B200LossWrapper(use_ppo=1) over an old-policy checkpoint: out has the reference's keys, loss.backward() sets every param.grad, the old
    policy's weights stay as loaded, and the step's scores are out['reward']."""
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    cfg = RNN_CFG
    B, n = 3, 4
    model = _engine('updown', cfg, _weights('updown', cfg))
    old_sd = {k: v.cuda() for k, v in _weights('updown', cfg, PERTURB['updown']).items()}
    path = str(tmp_path / 'old.pth')
    if lightning:
        torch.save({'pytorch-lightning_version': '1.5.0', 'state_dict': dict(old_sd, _vocab={'1': 'w1'}, _opt=argparse.Namespace(x=1))}, path)
    else:
        torch.save(old_sd, path)
    fc, att = co.make_inputs(B, R_FEATS, cfg['F_fc'], cfg['F_att'], seed=4)
    gts = cdo.make_refs(B, cfg['V'], seed=2)
    df, ref_len, table = _scorer(cfg)
    b200.rewards.reset_scorer()
    b200.rewards.init_scorer(table)
    try:
        lw = b200.B200LossWrapper(model, _lw_opt(n, path, w))
        frozen = {k: v.clone() for k, v in lw.old_model.state_dict().items()}
        labels = torch.zeros(B, n, cfg['T'] + 2, dtype=torch.long)
        labels[..., 1:4] = torch.randint(1, cfg['V'] + 1, (B, n, 3))
        masks = torch.zeros_like(labels, dtype=torch.float32)
        masks[..., :5] = 1
        out = lw(fc.cuda(), att.cuda(), labels.cuda(), masks.cuda(), None, gts, torch.arange(B), False, True, False)
        assert set(out) == {'loss', 'lm_loss', 'struc_loss', 'reward', 'pg_loss', 'kl_loss', 'clipfrac'}
        out['loss'].backward()
        torch.cuda.synchronize()
        assert all(p.grad is not None for p in model.parameters())
        for k, v in lw.old_model.state_dict().items():
            assert torch.equal(v, frozen[k]) and torch.equal(v, old_sd[k]), k
        seq = lw.last_step['sample_seq'].cpu().numpy()
        want = bo.get_scores(gts, seq, (1.0, 0.0), df, ref_len).astype(np.float32).reshape(B, n)
        assert out['reward'].shape == (B, n) and np.abs(out['reward'].cpu().numpy() - want).max() < 1e-5
        assert 0.0 <= float(out['clipfrac']) <= 1.0
    finally:
        b200.rewards.reset_scorer()
