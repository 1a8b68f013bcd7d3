"""The autograd path of the engine models (model.autograd) on the H100, for all five families in both parity modes: eval-mode gradients of a
random upstream dL/dlogprobs against torch autograd through the CPU oracle (teacher and sampling form), train mode with dropout against the
fused xe_step / scst_step under the same torch.manual_seed, an objective the fused steps refuse (the 'risk' structure loss), and the
interplay with the fused path (direct_grads views, accumulation, in-place weight updates, the flag off)."""
import pytest
import torch

import att2in2_oracle as ao
from helpers import LOGP_TOL, PARITY_MODES, co, family_opt

pytestmark = pytest.mark.gpu

GRAD_REL = 5e-4       # eval-mode parity with the oracle: every gradient within 5e-4 of the tensor's largest entry
FUSED_REL = 1e-5      # train mode against the fused steps (same kernels, same masks)
FAMILIES = ['updown', 'att2in2', 'newfc', 'aoa', 'transformer']
CFGS = {'updown': dict(V=40, E=32, H=48, A=24, F_fc=40, F_att=40, T=9),
        'att2in2': dict(V=40, E=32, H=48, A=24, F_fc=32, F_att=40, T=9),
        'newfc': dict(V=40, E=32, H=48, A=24, F_fc=40, F_att=40, T=9),
        'aoa': dict(V=40, E=32, H=64, A=0, F_fc=32, F_att=40, T=7),
        'transformer': dict(V=40, E=32, H=64, A=2, F_fc=32, F_att=40, T=7)}
HEADS = {'aoa': 8, 'transformer': 4}


def _setup(family, mode, seed=31, logit_scale=5.0):
    import imagecaptioning.pytorch_b200 as b200
    c = CFGS[family]
    dims = (c['V'], c['E'], c['H'], c['A'], c['F_fc'], c['F_att'])
    W = co.make_weights(family, *dims, seed=seed, logit_scale=logit_scale)
    opt = family_opt(family, *dims, c['T'], heads=HEADS.get(family, 8))
    opt.b200_autograd = 1
    m = b200.setup(opt, numeric_mode=mode)
    m.load_state_dict(W, strict=True)
    return m.cuda().eval(), W


def _oracle(family, W, requires_grad=True):
    Wg = {k: v.clone().requires_grad_(requires_grad and v.is_floating_point()) for k, v in W.items()}
    T = CFGS[family]['T']
    fam = ao.Att2in2Family(Wg, T) if family == 'att2in2' else co.Family(family, Wg, T, heads=HEADS.get(family, 8))
    return fam, Wg


def _inputs(family, B, R=6, seed=4):
    c = CFGS[family]
    fc, att = co.make_inputs(B, R, c['F_fc'], c['F_att'], seed=seed)
    if family == 'newfc':
        return fc, fc.new_zeros(B, 0, 0), None
    masks = torch.ones(B, R)
    masks[1, 4:] = 0
    return fc, att, masks


def _cuda(x):
    return None if x is None else x.cuda()


def _labels(B, spi, V, L, seed):
    g = torch.Generator().manual_seed(seed)
    labels = torch.zeros(B, spi, L, dtype=torch.long)
    masks = torch.zeros(B, spi, L)
    for i in range(B):
        for j in range(spi):
            n = int(torch.randint(2, L - 3, (1,), generator=g))      # every caption shorter than L - 2: the reference stops early
            labels[i, j, 1:1 + n] = torch.randint(1, V + 1, (n,), generator=g)
            masks[i, j, :n + 2] = 1
    return labels, masks


def _named_grads(model):
    return {k: p.grad for k, p in model.state_dict(keep_vars=True).items() if isinstance(p, torch.nn.Parameter)}


def _check(model, ograds, rel):
    got = _named_grads(model)
    assert got, 'no parameter gradients'
    largest = max(float(ograds[k].abs().max()) for k in got)
    for k, g in got.items():
        ref = ograds[k]
        assert g is not None, k
        scale = float(ref.abs().max())
        err = float((g.cpu() - ref).abs().max())
        # rel of the tensor's largest entry; tensors whose true gradient is zero (alpha_net.bias, and the attention key biases: softmax shift
        # invariance) hold rounding noise only and are held to 1e-5 of the largest gradient of the model
        assert err <= rel * scale + 1e-5 * largest, (k, err, scale, largest)
    assert sum(float(ograds[k].abs().max()) > 1e-3 * largest for k in got) >= 3      # the comparison is not vacuous


@pytest.mark.parametrize('mode', PARITY_MODES)
@pytest.mark.parametrize('family', FAMILIES)
def test_teacher_eval_parity(family, mode):
    """Teacher form, eval mode, seq_per_img 2 and region masks: engine gradients of a random upstream gradient against oracle autograd."""
    model, W = _setup(family, mode)
    B, spi, T = 3, 2, CFGS[family]['T']
    V = CFGS[family]['V']
    fc, att, masks = _inputs(family, B)
    labels, _ = _labels(B, spi, V, T + 2, seed=7)
    seq = labels[..., :-1]
    G = torch.randn(B * spi, T + 1, V + 1, generator=torch.Generator().manual_seed(3))
    lp = model(fc.cuda(), att.cuda(), seq.cuda(), _cuda(masks))
    assert lp.grad_fn is not None
    with torch.no_grad():
        plain = model(fc.cuda(), att.cuda(), seq.cuda(), _cuda(masks))
    assert plain.grad_fn is None
    assert float((lp.detach() - plain).abs().max()) < LOGP_TOL
    (lp * G.cuda()).sum().backward()
    fam, Wg = _oracle(family, W)
    olp = co.forward_teacher(fam, fc, att, seq, masks)
    assert float((lp.detach().cpu() - olp.detach()).abs().max()) < LOGP_TOL
    (olp * G).sum().backward()
    _check(model, {k: v.grad for k, v in Wg.items()}, GRAD_REL)
    if family != 'transformer':           # the reference's early stop: columns past it carry no log-probs and no gradient
        steps = model._teacher_steps(seq.reshape(B * spi, -1))
        assert steps < T + 1 and float(lp.detach()[:, steps:].abs().max()) == 0.0


@pytest.mark.parametrize('mode', PARITY_MODES)
@pytest.mark.parametrize('method,sample_n', [('greedy', 1), ('sample', 3)])
@pytest.mark.parametrize('family', FAMILIES)
def test_sample_eval_parity(family, mode, method, sample_n):
    """Sampling form, eval mode: the oracle replays the returned words; log-probs and gradients match."""
    model, W = _setup(family, mode, logit_scale=3.0)
    B, V = 3, CFGS[family]['V']
    fc, att, masks = _inputs(family, B)
    torch.manual_seed(5)
    seq, lp = model(fc.cuda(), att.cuda(), _cuda(masks), opt={'sample_method': method, 'sample_n': sample_n, 'beam_size': 1}, mode='sample')
    assert seq.shape == (B * sample_n, CFGS[family]['T']) and lp.grad_fn is not None
    G = torch.randn(lp.shape, generator=torch.Generator().manual_seed(9))
    (lp * G.cuda()).sum().backward()
    fam, Wg = _oracle(family, W)
    oseq, olp = co.sample(fam, fc, att, masks, sample_n=sample_n, forced_tokens=seq.cpu())
    assert torch.equal(oseq, seq.cpu())
    assert float((lp.detach().cpu() - olp.detach()).abs().max()) < LOGP_TOL
    (olp * G).sum().backward()
    _check(model, {k: v.grad for k, v in Wg.items()}, GRAD_REL)


def _fused_xe(model, fc, att, labels, masks, am, smoothing):
    kw = {'label_smoothing': smoothing, 'att_masks': am}
    res = model.xe_step(fc, att, labels, masks, **kw)
    return {k: res['grads'][p].clone() for k, p in model.state_dict(keep_vars=True).items() if p in res['grads']}


@pytest.mark.parametrize('mode', PARITY_MODES)
@pytest.mark.parametrize('family,smoothing,ss_prob', [('updown', 0.0, 0.0), ('updown', 0.2, 0.25), ('att2in2', 0.2, 0.0), ('newfc', 0.0, 0.0),
                                                      ('aoa', 0.0, 0.25), ('aoa', 0.2, 0.0), ('transformer', 0.0, 0.0), ('transformer', 0.2, 0.0)])
def test_train_xe_matches_fused_step(family, mode, smoothing, ss_prob):
    """Train mode, dropout on: LanguageModelCriterion / LabelSmoothing(0.2) on model(fc, att, labels[..., :-1]) give xe_step's gradients."""
    model, _ = _setup(family, mode)
    model.train()
    model.ss_prob = ss_prob
    B, spi, T, V = 3, 2, CFGS[family]['T'], CFGS[family]['V']
    fc, att, am = _inputs(family, B)
    labels, masks = _labels(B, spi, V, T + 2, seed=11)
    fc, att, am, labels, masks = fc.cuda(), att.cuda(), _cuda(am), labels.cuda(), masks.cuda()
    torch.manual_seed(123)
    ref = _fused_xe(model, fc, att, labels, masks, am, smoothing)
    torch.manual_seed(123)
    lp = model(fc, att, labels[..., :-1], am)
    if smoothing:
        loss = co.label_smoothing_loss(lp.cpu(), labels[..., 1:].cpu(), masks[..., 1:].cpu(), smoothing)
    else:
        loss = co.language_model_criterion(lp.cpu(), labels[..., 1:].cpu(), masks[..., 1:].cpu())
    loss.backward()
    _check(model, {k: v.cpu() for k, v in ref.items()}, FUSED_REL)


@pytest.mark.parametrize('mode', PARITY_MODES)
@pytest.mark.parametrize('family', FAMILIES)
def test_train_sampling_matches_scst_step(family, mode):
    """Train mode: the autograd _sample draws scst_step's words, and the leave-one-out reward of those draws (the engine's CIDEr-D scores
    through new_self_critical) gives scst_step(baseline='leave_one_out')'s gradients."""
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    model, _ = _setup(family, mode, logit_scale=3.0)
    model.train()
    B, n, V = 3, 3, CFGS[family]['V']
    fc, att, am = _inputs(family, B)
    fc, att, am = fc.cuda(), att.cuda(), _cuda(am)
    gts = cdo.make_refs(B, V, seed=2)
    df, ref_len = cdo.build_document_frequency(cdo.make_refs(50, V, seed=3))
    table = b200.rewards.CiderDTable(df, ref_len)
    torch.manual_seed(77)
    res = model.scst_step(fc, att, gts, table, n, baseline='leave_one_out', att_masks=am)
    ref = {k: res['grads'][p].clone().cpu() for k, p in model.state_dict(keep_vars=True).items() if p in res['grads']}
    fused_seq, reward = res['sample_seq'].clone(), res['reward'].clone()
    torch.manual_seed(77)
    seq, lp = model(fc, att, am, opt={'sample_method': 'sample', 'sample_n': n, 'beam_size': 1}, mode='sample')
    assert torch.equal(seq, fused_seq)
    # reward[n, t] is the row's leave-one-out advantage (constant over t): new_self_critical_loss of the scores it came from
    loss = co.reward_criterion(lp.cpu(), seq.cpu(), reward.cpu())
    loss.backward()
    _check(model, ref, FUSED_REL)


def _risk_loss(logprobs, seq, scores, n):
    """StructureLosses 'risk' (captioning/modules/losses.py:95-101), restated: the expected cost under the renormalised distribution of
    the n samples of each image, cost = -score."""
    mask = torch.cat([torch.ones(seq.shape[0], 1), (seq > 0).to(logprobs)[:, :-1]], 1)
    seq_lp = (logprobs.gather(2, seq.unsqueeze(2)).squeeze(2) * mask).sum(1) / mask.sum(1)
    probs = torch.softmax(seq_lp.view(-1, n), 1)
    return (probs * -scores.view(-1, n)).sum(1).mean()


@pytest.mark.parametrize('family', ['updown', 'transformer'])
def test_refused_objective_trains(family):
    """The 'risk' structure loss, which the fused steps refuse, trains through the autograd path: gradients match oracle autograd."""
    model, W = _setup(family, 'tc_f16x3', logit_scale=3.0)
    B, n = 3, 4
    fc, att, masks = _inputs(family, B)
    torch.manual_seed(8)
    seq, lp = model(fc.cuda(), att.cuda(), _cuda(masks), opt={'sample_method': 'sample', 'sample_n': n, 'beam_size': 1}, mode='sample')
    scores = torch.rand(B * n, generator=torch.Generator().manual_seed(1))
    _risk_loss(lp.cpu(), seq.cpu(), scores, n).backward()
    fam, Wg = _oracle(family, W)
    _, olp = co.sample(fam, fc, att, masks, sample_n=n, forced_tokens=seq.cpu())
    _risk_loss(olp, seq.cpu(), scores, n).backward()
    _check(model, {k: v.grad for k, v in Wg.items()}, GRAD_REL)


def test_fused_step_unaffected_by_autograd_in_between():
    """A fused step's gradients, delivered as direct_grads views of the flat buffer, are bit-identical whether or not an autograd forward
    and backward ran between its forward and its loss.backward()."""
    import argparse
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    B, n, V = 3, 3, CFGS['updown']['V']
    fc, att, am = _inputs('updown', B)
    fc, att, am = fc.cuda(), att.cuda(), am.cuda()
    gts = cdo.make_refs(B, V, seed=2)
    df, ref_len = cdo.build_document_frequency(cdo.make_refs(50, V, seed=3))
    b200.rewards.reset_scorer()
    b200.rewards.init_scorer(b200.rewards.CiderDTable(df, ref_len))
    opt = argparse.Namespace(sc_sample_method='greedy', sc_beam_size=1, train_sample_method='sample', train_beam_size=1, train_sample_n=n,
                             cider_reward_weight=1, bleu_reward_weight=0, label_smoothing=0.0, structure_loss_weight=1.0,
                             structure_loss_type='new_self_critical', use_ppo=0)
    labels, masks = _labels(B, 2, V, CFGS['updown']['T'] + 2, seed=3)
    model, _ = _setup('updown', 'tc_f16x3')
    model.train()
    lw = b200.B200LossWrapper(model, opt)            # direct_grads: param.grad become views of the flat buffer
    out = lw(fc, att, labels.cuda(), masks.cuda(), am, gts, torch.arange(B), False, True, False)
    flat = model._flat.flat
    fused = flat.clone()                             # the fused step wrote its gradients during its forward
    lp = model(fc, att, labels.cuda()[..., :-1], am)
    g = torch.autograd.grad(lp.sum(), list(model.parameters()))
    assert all(torch.isfinite(x).all() and float(x.abs().max()) > 0 for x in g)
    out['loss'].backward()
    b200.rewards.reset_scorer()
    assert torch.equal(flat, fused)
    base, end = flat.data_ptr(), flat.data_ptr() + flat.numel() * 4
    for p in model.parameters():
        assert base <= p.grad.data_ptr() < end        # still the views of the flat buffer


def test_accumulation_version_check_and_flag_off():
    model, _ = _setup('updown', 'tc_f16x3')
    B, spi, T, V = 3, 2, CFGS['updown']['T'], CFGS['updown']['V']
    fc, att, masks = _inputs('updown', B)
    fc, att, masks = fc.cuda(), att.cuda(), masks.cuda()
    seq = _labels(B, spi, V, T + 2, seed=5)[0][..., :-1].cuda()
    G = torch.randn(B * spi, T + 1, V + 1, device='cuda')
    lp = model(fc, att, seq, masks)
    (lp * G).sum().backward(retain_graph=True)
    once = [p.grad.clone() for p in model.parameters()]
    (lp * G).sum().backward()
    for p, g in zip(model.parameters(), once):
        assert torch.allclose(p.grad, 2 * g, rtol=0, atol=1e-6 * float(g.abs().max()) + 1e-12)
    # an in-place weight update between forward and backward raises torch's version error
    lp = model(fc, att, seq, masks)
    with torch.no_grad():
        model.logit.weight.add_(0.01)
    with pytest.raises(RuntimeError, match='modified by an inplace operation'):
        lp.sum().backward()
    # flag off: today's outputs, no grad_fn
    model.autograd = False
    plain = model(fc, att, seq, masks)
    with torch.no_grad():
        ref = model(fc, att, seq, masks)
    assert plain.grad_fn is None and torch.equal(plain, ref)
    s1, l1 = model(fc, att, masks, opt={'sample_method': 'greedy'}, mode='sample')
    assert l1.grad_fn is None
