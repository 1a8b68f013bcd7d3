"""Training with a vocabulary above 51 199 words (V = 60 000: V + 1 is odd, so the vocabulary step runs on a thread-block cluster and the
log-softmax backward, the XE / label-smoothing and SCST gradient kernels take their scalar paths) for all five families, against torch
autograd through the CPU oracle, dropout off:

* the fused XE step (LanguageModelCriterion and LabelSmoothing 0.2),
* the fused self-critical step with the oracle's draws replayed (samples and greedy baseline),
* the fused new_self_critical step (leave-one-out baseline) with the oracle's draws replayed,
* the autograd path (b200_autograd = 1): a teacher-forced backward of a random upstream gradient,
* one B200AttEnsemble greedy and sampling call.

Loss and reward within 1e-4; every gradient within 5e-4 of its tensor's largest entry (tensors whose true gradient is zero: 1e-5 of the
model's largest gradient)."""
import numpy as np
import pytest
import torch

import att2in2_oracle as ao
import ensemble_oracle as eo
from helpers import LOGP_TOL, check_decode, co, family_opt

pytestmark = pytest.mark.gpu

V = 60000
FAMILIES = ['updown', 'att2in2', 'newfc', 'aoa', 'transformer']
CFGS = {'updown': dict(E=32, H=32, A=16, F_fc=40, F_att=40, T=9),
        'att2in2': dict(E=32, H=32, A=16, F_fc=40, F_att=40, T=9),
        'newfc': dict(E=32, H=32, A=16, F_fc=40, F_att=40, T=9),
        'aoa': dict(E=32, H=32, A=0, F_fc=32, F_att=40, T=7),
        'transformer': dict(E=32, H=64, A=2, F_fc=32, F_att=40, T=7)}
HEADS = {'aoa': 4, 'transformer': 4}
NO_DROPOUT = {'updown': dict(drop_prob=0.0), 'att2in2': dict(drop_prob=0.0), 'newfc': dict(drop_prob=0.0),
              'aoa': dict(drop_prob=0.0, drop_attn=0.0, drop_aoa=0.0, drop_sublayer=0.0), 'transformer': dict(drop_prob=0.0, dropout=0.0)}
GRAD_REL = 5e-4
B, R = 3, 6


def _dims(family):
    c = CFGS[family]
    return (V, c['E'], c['H'], c['A'], c['F_fc'], c['F_att'])


def _model(family, seed=31, logit_scale=3.0, autograd=False):
    import imagecaptioning.pytorch_b200 as b200
    W = co.make_weights(family, *_dims(family), seed=seed, logit_scale=logit_scale)
    opt = family_opt(family, *_dims(family), CFGS[family]['T'], heads=HEADS.get(family, 8))
    if autograd:
        opt.b200_autograd = 1
    m = b200.setup(opt, numeric_mode='tc_f16x3')
    m.load_state_dict(W, strict=True)
    return m.cuda(), W


def _oracle(family, W):
    Wg = {k: v.clone().requires_grad_(v.is_floating_point()) for k, v in W.items()}
    T = CFGS[family]['T']
    fam = ao.Att2in2Family(Wg, T) if family == 'att2in2' else co.Family(family, Wg, T, heads=HEADS.get(family, 8))
    return fam, Wg


def _inputs(family, seed=4):
    c = CFGS[family]
    fc, att = co.make_inputs(B, R, c['F_fc'], c['F_att'], seed=seed)
    if family == 'newfc':
        att = fc.new_zeros(B, 0, 0)
    return fc, att


def _table(B):
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    gts = cdo.make_refs(B, V, seed=2)
    df, ref_len = cdo.build_document_frequency(cdo.make_refs(50, V, seed=3))
    return gts, b200.rewards.CiderDTable(df, ref_len), df, ref_len


def _labels(spi, L, seed):
    g = torch.Generator().manual_seed(seed)
    labels = torch.zeros(B, spi, L, dtype=torch.long)
    masks = torch.zeros(B, spi, L)
    for i in range(B):
        for j in range(spi):
            n = int(torch.randint(2, L - 3, (1,), generator=g))
            labels[i, j, 1:1 + n] = torch.randint(1, V + 1, (n,), generator=g)
            masks[i, j, :n + 2] = 1
    return labels, masks


def _check_grads(model, grads, Wg):
    """grads: {parameter: gradient} of the engine; Wg: the oracle's weights after backward()."""
    name_of = {id(p): k for k, p in model.state_dict(keep_vars=True).items()}
    named = {name_of[id(p)]: g for p, g in grads.items()}
    assert named, 'no parameter gradients'
    largest = max(float(Wg[k].grad.abs().max()) for k in named)
    assert largest > 0
    for k, g in named.items():
        ref = Wg[k].grad
        err = float((g.cpu() - ref).abs().max())
        assert err <= GRAD_REL * float(ref.abs().max()) + 1e-5 * largest, (k, err, float(ref.abs().max()), largest)
    for k in ('logit.weight', 'model.generator.proj.weight'):
        if k in named:
            assert float(Wg[k].grad.abs().max()) > 1e-3 * largest          # the [V+1, .] gradients are not vacuous


@pytest.mark.parametrize('smoothing', [0.0, 0.2])
@pytest.mark.parametrize('family', FAMILIES)
def test_xe_step(family, smoothing):
    model, W = _model(family)
    model.train()
    T = CFGS[family]['T']
    fc, att = _inputs(family)
    labels, masks = _labels(2, T + 2, seed=11)
    res = model.xe_step(fc.cuda(), att.cuda(), labels.cuda(), masks.cuda(), label_smoothing=smoothing, seed=1, **NO_DROPOUT[family])
    torch.cuda.synchronize()
    fam, Wg = _oracle(family, W)
    lp = co.forward_teacher(fam, fc, att, labels[..., :-1], pad_keys_masked=True)
    if smoothing:
        loss = co.label_smoothing_loss(lp, labels[..., 1:], masks[..., 1:], smoothing)
    else:
        loss = co.language_model_criterion(lp, labels[..., 1:], masks[..., 1:])
    loss.backward()
    assert res['logprobs'].shape[-1] == V + 1
    assert abs(float(res['loss']) - float(loss)) < LOGP_TOL, (float(res['loss']), float(loss))
    _check_grads(model, res['grads'], Wg)


@pytest.mark.parametrize('baseline', ['greedy', 'leave_one_out'])
@pytest.mark.parametrize('family', FAMILIES)
def test_scst_and_new_self_critical_steps_replaying_the_oracle_draws(family, baseline):
    """The oracle draws the samples (and the greedy baseline); the fused step replays them.  'greedy' is the self-critical step,
    'leave_one_out' the new_self_critical structure loss."""
    from oracle import ciderd_oracle as cdo
    model, W = _model(family, logit_scale=5.0)
    model.train()
    n = 4
    fc, att = _inputs(family)
    gts, table, df, ref_len = _table(B)
    fam0, _ = _oracle(family, W)
    torch.manual_seed(3)
    with torch.no_grad():
        o_base, _ = co.sample(fam0, fc, att)
        o_seq, _ = co.sample(fam0, fc, att, sample_method='sample', sample_n=n)
    # words drawn from 60 000 share no n-gram with the synthetic references: each image's first sample joins its references, so that
    # the rewards, the loss and the gradients are not all zero
    T = o_seq.shape[1]
    gts = [np.concatenate([g, np.pad(o_seq[i * n].numpy(), (0, g.shape[1] - T))[None]]) for i, g in enumerate(gts)]
    kw = dict(forced_tokens=o_seq.cuda(), seed=1, baseline=baseline, **NO_DROPOUT[family])
    if baseline == 'greedy':
        kw['forced_baseline'] = o_base.cuda()
    res = model.scst_step(fc.cuda(), att.cuda(), gts, table, n, **kw)
    torch.cuda.synchronize()
    assert torch.equal(res['sample_seq'].cpu(), o_seq)
    fam, Wg = _oracle(family, W)
    _, lp = co.sample(fam, fc, att, sample_method='sample', sample_n=n, forced_tokens=o_seq)
    assert float((res['sample_logprobs'].cpu() - lp.detach()).abs().max()) < LOGP_TOL
    if baseline == 'greedy':
        assert torch.equal(res['greedy_seq'].cpu(), o_base)
        reward, _ = cdo.self_critical_reward(o_base.numpy(), gts, o_seq.numpy(), df, ref_len)
        reward = torch.from_numpy(reward).float()
        loss = co.reward_criterion(lp, o_seq, reward)
        assert float((res['reward'].cpu() - reward).abs().max()) < LOGP_TOL
    else:
        scores = torch.from_numpy(cdo.get_scores(gts, o_seq.numpy(), df, ref_len)).float()
        s = scores.double().reshape(B, n)
        advantage = (s - (s.sum(1, keepdim=True) - s) / (n - 1)).reshape(-1, 1).expand(-1, T)      # losses.py:168-187
        assert float((res['reward'].cpu().double() - advantage).abs().max()) < LOGP_TOL
        loss = co.new_self_critical_loss(lp, o_seq, scores, n)
    loss.backward()
    assert abs(float(res['loss']) - float(loss)) < LOGP_TOL and abs(float(loss)) > 1e-4, (float(res['loss']), float(loss))
    _check_grads(model, res['grads'], Wg)


def test_autograd_teacher_backward():
    """b200_autograd = 1: model(fc, att, labels) under grad, backward of a random upstream gradient, against oracle autograd."""
    family = 'updown'
    model, W = _model(family, logit_scale=5.0, autograd=True)
    model.eval()
    T = CFGS[family]['T']
    fc, att = _inputs(family)
    labels, _ = _labels(2, T + 2, seed=7)
    seq = labels[..., :-1]
    lp = model(fc.cuda(), att.cuda(), seq.cuda(), None)
    assert lp.grad_fn is not None and lp.shape[-1] == V + 1
    G = torch.randn(lp.shape, generator=torch.Generator().manual_seed(3))
    (lp * G.cuda()).sum().backward()
    fam, Wg = _oracle(family, W)
    olp = co.forward_teacher(fam, fc, att, seq)
    assert float((lp.detach().cpu().reshape(olp.shape) - olp.detach()).abs().max()) < LOGP_TOL
    (olp * G.reshape(olp.shape)).sum().backward()
    grads = {p: p.grad for p in model.parameters() if p.grad is not None}
    _check_grads(model, grads, Wg)


def test_ensemble_greedy_and_sampling():
    """B200AttEnsemble of an UpDown and an Att2in2 member at V = 60 000: greedy ids bit-exact and log-probs within 1e-4 against the oracle's
    mixture, and a sampling call whose rows are the oracle's mixture rows of the drawn words."""
    import imagecaptioning.pytorch_b200 as b200
    members, ofams = [], []
    for family, seed in (('updown', 5), ('att2in2', 6)):
        c = CFGS[family]
        W = co.make_weights(family, *_dims(family), seed=seed, logit_scale=8.0)
        m = b200.setup(family_opt(family, *_dims(family), c['T']), numeric_mode='tc_f16x3')
        m.load_state_dict(W, strict=True)
        members.append(m.cuda().eval())
        ofams.append(eo.member_family(family, W, c['T']))
    ens = b200.B200AttEnsemble(members, weights=[0.7, 0.3])
    ofam = eo.EnsembleFamily(ofams, [0.7, 0.3])
    fc, att = co.make_inputs(B, R, 40, 40, seed=9)
    with torch.no_grad():
        seq, lp = ens(fc.cuda(), att.cuda(), None, opt={'sample_method': 'greedy', 'beam_size': 1}, mode='sample')
        margins = []
        oseq, olp = co.sample(ofam, fc, att, record_margin=margins)
        assert lp.shape[-1] == V + 1
        assert check_decode(ofam, fc, att, seq, lp, oseq, olp, margins), min(margins)
        torch.manual_seed(2)
        seq, lp = ens(fc.cuda(), att.cuda(), None, opt={'sample_method': 'sample', 'sample_n': 3, 'beam_size': 1}, mode='sample')
        _, olp = co.sample(ofam, fc, att, sample_n=3, forced_tokens=seq.cpu())
        assert float((lp.cpu() - olp).abs().max()) < LOGP_TOL
        assert len(set(seq.cpu().reshape(-1).tolist())) > 3
