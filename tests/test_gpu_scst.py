"""GPU parity of the SCST training step (UpDown): loss, reward and every parameter gradient against torch autograd through the
oracle on the CPU, with the engine's own samples and (when dropout is on) its own dropout masks replayed in the oracle."""
import argparse

import numpy as np
import pytest
import torch

from helpers import LOGP_TOL, aoa_masks, build_pair, co, dropout_masks

pytestmark = pytest.mark.gpu

CFG = dict(V=40, E=32, H=48, A=24, F_fc=32, F_att=40, T=9)


def _oracle_grads(W, fc, att, gts, df, ref_len, sample_seq, greedy_seq, n, drop):
    from oracle import ciderd_oracle as cdo
    Wg = {k: v.clone().requires_grad_(True) for k, v in W.items()}
    fam = co.Family('updown', Wg, CFG['T'])
    fam.drop = drop
    _, lp = co.sample(fam, fc, att, sample_method='sample', sample_n=n, forced_tokens=sample_seq)
    reward, _ = cdo.self_critical_reward(greedy_seq.numpy(), gts, sample_seq.numpy(), df, ref_len)
    reward = torch.from_numpy(reward).float()
    loss = co.reward_criterion(lp, sample_seq, reward)
    loss.backward()
    return float(loss), reward, {k: v.grad for k, v in Wg.items()}, lp.detach()


@pytest.mark.parametrize('drop_prob', [0.0, 0.5])
@pytest.mark.parametrize('mode', ['tc_f16x3', 'simt_fp32'])
def test_scst_step_gradients(mode, drop_prob):
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    model, fam = build_pair('updown', seed=31, logit_scale=5.0, mode=mode, **CFG)
    W = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    B, R, n, T = 5, 11, 4, CFG['T']
    fc, att = co.make_inputs(B, R, CFG['F_fc'], CFG['F_att'], seed=4)
    gts = cdo.make_refs(B, CFG['V'], seed=2)
    df, ref_len = cdo.build_document_frequency(cdo.make_refs(200, CFG['V'], seed=4))
    table = b200.rewards.CiderDTable(df, ref_len)
    model.train()
    res = model.scst_step(fc.cuda(), att.cuda(), gts, table, n, temperature=1.0, drop_prob=drop_prob, seed=1234)
    torch.cuda.synchronize()
    sample_seq, greedy_seq = res['sample_seq'].cpu(), res['greedy_seq'].cpu()
    # greedy baseline = eval-mode greedy decode of the oracle
    og, _ = co.sample(fam, fc, att)
    assert torch.equal(greedy_seq, og)
    drop = None
    if drop_prob > 0:
        L, lib = b200._lib, b200._lib.load()
        N, E, H = B * n, CFG['E'], CFG['H']

        def mask(site, step, rows, cols):
            m = torch.empty(rows * cols, device='cuda')
            L.check(lib.capb200_dropout_mask(L.ptr(m), rows * cols, 1234, site, step, drop_prob, L.current_stream()), 'dropout_mask')
            return m.cpu().reshape(rows, cols)
        drop = {'fc': mask(0, 0, B, H), 'att': mask(1, 0, B * R, H).reshape(B, R, H),
                'xt': torch.stack([mask(2, t, N, E) for t in range(T)]), 'out': torch.stack([mask(3, t, N, H) for t in range(T)])}
        keep = float((drop['att'] > 0).float().mean())
        assert abs(keep - (1 - drop_prob)) < 0.03 and abs(float(drop['att'].max()) - 1 / (1 - drop_prob)) < 1e-6
    oloss, oreward, ograds, olp = _oracle_grads(W, fc, att, gts, df, ref_len, sample_seq, greedy_seq, n, drop)
    assert float((res['sample_logprobs'].cpu() - olp).abs().max()) < LOGP_TOL
    assert float((res['reward'].cpu() - oreward).abs().max()) < LOGP_TOL
    assert abs(float(res['loss']) - oloss) < LOGP_TOL
    name_of = {id(p): k for k, p in model.state_dict(keep_vars=True).items()}
    worst = 0.0
    for p, g in res['grads'].items():
        key = name_of[id(p)]
        ref = ograds[key]
        scale = float(ref.abs().max())
        err = float((g.cpu() - ref).abs().max())
        if scale > 1e-7:
            worst = max(worst, err / scale)
        assert err <= 5e-4 * scale + 2e-9, (key, err, scale)      # 5e-4 of the tensor's largest gradient entry
    assert abs(oloss) > 1e-2 and sum(float(v.abs().max()) > 1e-5 for v in ograds.values()) >= 15      # the comparison is not vacuous
    print('max relative gradient error', worst)


def test_loss_wrapper_backward_sets_param_grads():
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    model, _ = build_pair('updown', seed=31, logit_scale=5.0, mode='tc_f16x3', **CFG)
    B, R, n = 4, 7, 3
    fc, att = co.make_inputs(B, R, CFG['F_fc'], CFG['F_att'], seed=5)
    gts = cdo.make_refs(B, CFG['V'], seed=3)
    df, ref_len = cdo.build_document_frequency(cdo.make_refs(100, CFG['V'], seed=4))
    b200.rewards.reset_scorer()
    b200.rewards.init_scorer(b200.rewards.CiderDTable(df, ref_len))
    opt = argparse.Namespace(sc_sample_method='greedy', sc_beam_size=1, train_sample_method='sample', train_beam_size=1, train_sample_n=n,
                             cider_reward_weight=1, bleu_reward_weight=0)
    lw = b200.B200LossWrapper(model, opt)
    out = lw(fc.cuda(), att.cuda(), None, None, None, gts, torch.arange(B), True, False, False)
    assert out['loss'].requires_grad
    step = lw.last_step
    engine_grads = {p: g.clone() for p, g in step['grads'].items()}
    (2.0 * out['loss']).backward()
    for p, g in step['grads'].items():
        # direct path (default): the flat buffer was scaled in place by the upstream gradient and param.grad is a VIEW of it
        assert p.grad is not None and p.grad.data_ptr() == g.data_ptr() and torch.allclose(p.grad, 2.0 * engine_grads[p])
    # zero_grad(set_to_none=False) (the default of the torch versions the reference targets) keeps the views: the next step's gradients land in them
    model.zero_grad(set_to_none=False)
    out_b = lw(fc.cuda(), att.cuda(), None, None, None, gts, torch.arange(B), True, False, False)
    engine_grads = {p: g.clone() for p, g in lw.last_step['grads'].items()}
    out_b['loss'].backward()
    for p, g in lw.last_step['grads'].items():
        assert p.grad.data_ptr() == g.data_ptr() and torch.allclose(p.grad, engine_grads[p])
    # through autograd (what torch DDP / gradient accumulation need): fresh tensors, accumulated like any other gradient
    model.zero_grad(set_to_none=True)
    lw.direct_grads = False
    out_c = lw(fc.cuda(), att.cuda(), None, None, None, gts, torch.arange(B), True, False, False)
    engine_grads = {p: g.clone() for p, g in lw.last_step['grads'].items()}
    (3.0 * out_c['loss']).backward()
    for p, g in lw.last_step['grads'].items():
        assert p.grad.data_ptr() != g.data_ptr() and torch.allclose(p.grad, 3.0 * engine_grads[p])
    lw.direct_grads = True
    # an optimizer step changes the weights, the next call re-binds them (version counters) and still works
    torch.optim.SGD(model.parameters(), lr=1e-3).step()
    out2 = lw(fc.cuda(), att.cuda(), None, None, None, gts, torch.arange(B), True, False, False)
    assert torch.isfinite(out2['loss'])
    b200.rewards.reset_scorer()


def _check_grads(model, grads, ograds, rel=5e-4):
    name_of = {id(p): k for k, p in model.state_dict(keep_vars=True).items()}
    largest = max(float(v.abs().max()) for v in ograds.values())
    for p, g in grads.items():
        key = name_of[id(p)]
        ref = ograds[key]
        scale = float(ref.abs().max())
        err = float((g.cpu() - ref).abs().max())
        # 5e-4 of the tensor's largest entry; tensors whose true gradient is zero (alpha_net.bias: softmax shift invariance) are held to
        # 1e-7 of the largest gradient of the step
        assert err <= rel * scale + 1e-7 * largest, (key, err, scale)
    assert sum(float(v.abs().max()) > 1e-5 for v in ograds.values()) >= 15


def _labels(B, spi, V, cols, seed, short=False):
    g = torch.Generator().manual_seed(seed)
    labels = torch.zeros(B, spi, cols, dtype=torch.long)
    masks = torch.zeros(B, spi, cols)
    for i in range(B):
        for j in range(spi):
            ln = int(torch.randint(1, cols - (4 if short else 1), (1,), generator=g))
            labels[i, j, 1:1 + ln] = torch.randint(1, V + 1, (ln,), generator=g)
            masks[i, j, :ln + 2] = 1
    return labels, masks


@pytest.mark.parametrize('smoothing', [0.0, 0.1])
@pytest.mark.parametrize('mode,drop_prob,short', [('tc_f16x3', 0.0, False), ('tc_f16x3', 0.5, True), ('simt_fp32', 0.5, False)])
def test_xe_step_gradients(mode, drop_prob, short, smoothing):
    """Teacher-forced XE step (AttModel._forward + LanguageModelCriterion / LabelSmoothing + backward) against autograd through the
    oracle, with the engine's dropout masks replayed; ``short`` labels end early so the data-dependent break is exercised."""
    import imagecaptioning.pytorch_b200 as b200
    model, _ = build_pair('updown', seed=31, logit_scale=5.0, mode=mode, **CFG)
    W = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    B, R, spi, T = 4, 9, 3, CFG['T']
    fc, att = co.make_inputs(B, R, CFG['F_fc'], CFG['F_att'], seed=6)
    labels, masks = _labels(B, spi, CFG['V'], T + 2, seed=9, short=short)
    model.train()
    res = model.xe_step(fc.cuda(), att.cuda(), labels.cuda(), masks.cuda(), label_smoothing=smoothing, drop_prob=drop_prob, seed=77)
    torch.cuda.synchronize()
    Wg = {k: v.clone().requires_grad_(True) for k, v in W.items()}
    fam = co.Family('updown', Wg, T)
    if drop_prob > 0:
        fam.drop = dropout_masks(b200, 77, drop_prob, B, R, B * spi, T + 1, CFG['E'], CFG['H'])
    lp = co.forward_teacher(fam, fc, att, labels[..., :-1])
    if short:
        assert float(lp[:, -1].abs().max()) == 0.0
    tl, tm = labels[..., 1:].reshape(B * spi, -1), masks[..., 1:].reshape(B * spi, -1)
    loss = co.language_model_criterion(lp, tl, tm) if smoothing == 0 else co.label_smoothing_loss(lp, tl, tm, smoothing)
    loss.backward()
    assert float((res['logprobs'].cpu() - lp.detach()).abs().max()) < LOGP_TOL
    assert abs(float(res['loss']) - float(loss)) < LOGP_TOL
    _check_grads(model, res['grads'], {k: v.grad for k, v in Wg.items()})


def test_xe_step_matches_reference_golden():
    """The XE loss and parameter gradients the live reference produced (tests/golden/xe_struct.npz), straight against the engine."""
    import os
    g = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'xe_struct.npz'))
    V, E, H, A, F_fc, F_att, T, B, R, spi, seed = (int(x) for x in g['xe_cfg'])
    model, _ = build_pair('updown', V=V, E=E, H=H, A=A, F_fc=F_fc, F_att=F_att, T=T, seed=seed, logit_scale=20.0, mode='tc_f16x3')
    fc, att = co.make_inputs(B, R, F_fc, F_att, seed=seed)
    model.train()
    name_of = {id(p): k for k, p in model.state_dict(keep_vars=True).items()}
    for name, smoothing in (('xe', 0.0), ('xels', 0.1)):
        res = model.xe_step(fc.cuda(), att.cuda(), torch.from_numpy(g['xe_labels']).cuda(), torch.from_numpy(g['xe_masks']).cuda(),
                            label_smoothing=smoothing, drop_prob=0.0, seed=1)
        assert abs(float(res['loss']) - float(g[name + '_loss'])) < LOGP_TOL
        if smoothing == 0:
            assert np.abs(res['logprobs'].cpu().numpy() - g['xe_logprobs']).max() < LOGP_TOL
        checked = 0
        largest = max(float(np.abs(g[k]).max()) for k in g.files if k.startswith(name + '_grad_'))
        for p, grad in res['grads'].items():
            key = name + '_grad_' + name_of[id(p)]
            if key in g.files:
                ref = g[key]
                # alpha_net.bias has a mathematically zero gradient (softmax shift invariance): absolute floor relative to the step
                assert np.abs(grad.cpu().numpy() - ref).max() <= 5e-4 * np.abs(ref).max() + 1e-7 * largest, key
                checked += 1
        assert checked == 8


@pytest.mark.parametrize('drop_prob', [0.0, 0.5])
def test_new_self_critical_step(drop_prob):
    """Structure loss 'new_self_critical' (losses.py:168-187): leave-one-out CIDEr-D baseline, no greedy decode."""
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    model, _ = build_pair('updown', seed=31, logit_scale=5.0, mode='tc_f16x3', **CFG)
    W = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    B, R, n, T = 5, 11, 4, CFG['T']
    fc, att = co.make_inputs(B, R, CFG['F_fc'], CFG['F_att'], seed=4)
    gts = cdo.make_refs(B, CFG['V'], seed=2)
    df, ref_len = cdo.build_document_frequency(cdo.make_refs(200, CFG['V'], seed=4))
    table = b200.rewards.CiderDTable(df, ref_len)
    model.train()
    res = model.scst_step(fc.cuda(), att.cuda(), gts, table, n, drop_prob=drop_prob, seed=99, baseline='leave_one_out')
    torch.cuda.synchronize()
    assert res['greedy_seq'] is None
    seq = res['sample_seq'].cpu()
    Wg = {k: v.clone().requires_grad_(True) for k, v in W.items()}
    fam = co.Family('updown', Wg, T)
    if drop_prob > 0:
        fam.drop = dropout_masks(b200, 99, drop_prob, B, R, B * n, T, CFG['E'], CFG['H'])
    _, lp = co.sample(fam, fc, att, sample_method='sample', sample_n=n, forced_tokens=seq)
    scores = torch.from_numpy(cdo.get_scores(gts, seq.numpy(), df, ref_len))
    loss = co.new_self_critical_loss(lp, seq, scores, n)
    loss.backward()
    dev_scores = b200.rewards.cider_scores(gts, res['sample_seq'], table)
    assert float((dev_scores.cpu() - scores).abs().max()) < 1e-9
    sc = scores.float().view(B, n)
    adv = (sc - (sc.sum(1, keepdim=True) - sc) / (n - 1)).reshape(-1)
    assert float((res['reward'][:, 0].cpu() - adv).abs().max()) < LOGP_TOL
    assert abs(float(res['loss']) - float(loss)) < LOGP_TOL
    assert float(adv.abs().max()) > 1e-3
    _check_grads(model, res['grads'], {k: v.grad for k, v in Wg.items()})


def test_loss_wrapper_xe_and_structure_branches():
    """B200LossWrapper: sc_flag=False (XE) and struc_flag=True with structure_loss_weight in {1, 0.5} produce losses wired to autograd."""
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    model, _ = build_pair('updown', seed=31, logit_scale=5.0, mode='tc_f16x3', **CFG)
    B, R, n, spi, T = 4, 7, 3, 2, CFG['T']
    fc, att = co.make_inputs(B, R, CFG['F_fc'], CFG['F_att'], seed=5)
    labels, masks = _labels(B, spi, CFG['V'], T + 2, seed=3)
    gts = cdo.make_refs(B, CFG['V'], seed=3)
    df, ref_len = cdo.build_document_frequency(cdo.make_refs(100, CFG['V'], seed=4))
    b200.rewards.reset_scorer()
    b200.rewards.init_scorer(b200.rewards.CiderDTable(df, ref_len))
    opt = argparse.Namespace(sc_sample_method='greedy', sc_beam_size=1, train_sample_method='sample', train_beam_size=1, train_sample_n=n,
                             cider_reward_weight=1, bleu_reward_weight=0, label_smoothing=0.0, structure_loss_weight=1.0,
                             structure_loss_type='new_self_critical', use_ppo=0)
    lw = b200.B200LossWrapper(model, opt)
    model.train()
    args = (fc.cuda(), att.cuda(), labels.cuda(), masks.cuda(), None, gts, torch.arange(B))
    out = lw(*args, False, False, False)
    ref = lw.crit(model(fc.cuda(), att.cuda(), labels.cuda()[..., :-1], None), labels.cuda()[..., 1:], masks.cuda()[..., 1:])
    out['loss'].backward()
    assert all(p.grad is not None for p in model.parameters())
    assert torch.isfinite(ref) and float(ref) > 0                       # eval-mode teacher forcing of the engine + host criterion
    out = lw(*args, False, True, False)
    assert out['reward'].shape == (B, n) and float(out['lm_loss']) == 0.0 and out['loss'].requires_grad
    opt.structure_loss_weight = 0.5
    model.zero_grad()
    out = lw(*args, False, True, False)
    assert abs(float(out['loss']) - 0.5 * float(out['lm_loss']) - 0.5 * float(out['struc_loss'])) < 1e-6
    out['loss'].backward()
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in model.parameters())
    b200.rewards.reset_scorer()


AOA_CFG = dict(V=40, E=32, H=64, A=0, F_fc=32, F_att=40, T=7)


@pytest.mark.parametrize('mode,dropout,baseline', [('tc_f16x3', False, 'greedy'), ('tc_f16x3', True, 'greedy'), ('simt_fp32', True, 'leave_one_out')])
def test_aoa_scst_step_gradients(mode, dropout, baseline):
    """AoANet SCST step (BASELINE configs[3]): loss, reward and every parameter gradient against torch autograd through the oracle, with
    the engine's samples and all of its dropout masks (att_embed, refiner attention / AoA / sublayer, word, ctx, decoder attention,
    output) replayed in the oracle."""
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    heads = 4
    model, fam = build_pair('aoa', seed=21, logit_scale=5.0, mode=mode, heads=heads, **AOA_CFG)
    W = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    B, R, n, T = 3, 9, 3, AOA_CFG['T']
    E, H = AOA_CFG['E'], AOA_CFG['H']
    fc, att = co.make_inputs(B, R, AOA_CFG['F_fc'], AOA_CFG['F_att'], seed=4)
    gts = cdo.make_refs(B, AOA_CFG['V'], seed=2)
    df, ref_len = cdo.build_document_frequency(cdo.make_refs(200, AOA_CFG['V'], seed=4))
    table = b200.rewards.CiderDTable(df, ref_len)
    p_lm, p_at, p_aoa, p_sub = (0.5, 0.1, 0.3, 0.1) if dropout else (0.0, 0.0, 0.0, 0.0)
    model.train()
    res = model.scst_step(fc.cuda(), att.cuda(), gts, table, n, drop_prob=p_lm, seed=4321, baseline=baseline, drop_attn=p_at, drop_aoa=p_aoa,
                          drop_sublayer=p_sub, ctx_drop=1)
    torch.cuda.synchronize()
    seq = res['sample_seq'].cpu()
    Wg = {k: v.clone().requires_grad_(True) for k, v in W.items()}
    fam_g = co.Family('aoa', Wg, T, heads=heads)
    if dropout:
        fam_g.drop = aoa_masks(b200, 4321, B, R, B * n, T, E, H, heads, p_lm, p_at, p_aoa, p_sub)
    _, lp = co.sample(fam_g, fc, att, sample_method='sample', sample_n=n, forced_tokens=seq)
    if baseline == 'greedy':
        og, _ = co.sample(fam, fc, att)
        assert torch.equal(res['greedy_seq'].cpu(), og)
        reward, _ = cdo.self_critical_reward(og.numpy(), gts, seq.numpy(), df, ref_len)
        reward = torch.from_numpy(reward).float()
        loss = co.reward_criterion(lp, seq, reward)
    else:
        scores = torch.from_numpy(cdo.get_scores(gts, seq.numpy(), df, ref_len))
        loss = co.new_self_critical_loss(lp, seq, scores, n)
        sc = scores.float().view(B, n)
        reward = (sc - (sc.sum(1, keepdim=True) - sc) / (n - 1)).reshape(-1, 1).expand(-1, T)
    loss.backward()
    assert float((res['sample_logprobs'].cpu() - lp.detach()).abs().max()) < LOGP_TOL
    assert float((res['reward'].cpu() - reward).abs().max()) < LOGP_TOL
    assert abs(float(res['loss']) - float(loss)) < LOGP_TOL
    assert float(reward.abs().max()) > 1e-3                       # the comparison is not vacuous (the leave-one-out loss itself is ~0)
    _check_grads(model, res['grads'], {k: v.grad for k, v in Wg.items()})


@pytest.mark.parametrize('dropout,smoothing', [(False, 0.0), (True, 0.1)])
def test_aoa_xe_step_gradients(dropout, smoothing):
    """AoANet XE step: teacher-forced train-mode forward, LanguageModelCriterion / LabelSmoothing and every gradient against autograd
    through the oracle with the engine's dropout masks replayed (labels end early: the data-dependent break is exercised)."""
    import imagecaptioning.pytorch_b200 as b200
    heads = 4
    model, _ = build_pair('aoa', seed=21, logit_scale=5.0, mode='tc_f16x3', heads=heads, **AOA_CFG)
    W = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    B, R, spi, T = 3, 9, 2, AOA_CFG['T']
    E, H = AOA_CFG['E'], AOA_CFG['H']
    fc, att = co.make_inputs(B, R, AOA_CFG['F_fc'], AOA_CFG['F_att'], seed=4)
    labels, masks = _labels(B, spi, AOA_CFG['V'], T + 2, seed=12, short=True)
    p_lm, p_at, p_aoa, p_sub = (0.5, 0.1, 0.3, 0.1) if dropout else (0.0, 0.0, 0.0, 0.0)
    model.train()
    res = model.xe_step(fc.cuda(), att.cuda(), labels.cuda(), masks.cuda(), label_smoothing=smoothing, drop_prob=p_lm, seed=555, drop_attn=p_at,
                        drop_aoa=p_aoa, drop_sublayer=p_sub, ctx_drop=1)
    torch.cuda.synchronize()
    Wg = {k: v.clone().requires_grad_(True) for k, v in W.items()}
    fam = co.Family('aoa', Wg, T, heads=heads)
    if dropout:
        fam.drop = aoa_masks(b200, 555, B, R, B * spi, T + 1, E, H, heads, p_lm, p_at, p_aoa, p_sub)
    lp = co.forward_teacher(fam, fc, att, labels[..., :-1])
    assert float(lp[:, -1].abs().max()) == 0.0
    tl, tm = labels[..., 1:].reshape(B * spi, -1), masks[..., 1:].reshape(B * spi, -1)
    loss = co.language_model_criterion(lp, tl, tm) if smoothing == 0 else co.label_smoothing_loss(lp, tl, tm, smoothing)
    loss.backward()
    assert float((res['logprobs'].cpu() - lp.detach()).abs().max()) < LOGP_TOL
    assert abs(float(res['loss']) - float(loss)) < LOGP_TOL
    _check_grads(model, res['grads'], {k: v.grad for k, v in Wg.items()})


def test_cider_kernel_on_real_captions(golden_dir):
    """The CIDEr-D reward kernel on real text: 60 PASCAL-50S images with 50 references each (tests/golden/ciderd_pascal.npz, produced by
    the live reference scorer), document-frequency table of 38 k n-grams."""
    import os
    import imagecaptioning.pytorch_b200 as b200
    g = np.load(os.path.join(golden_dir, 'ciderd_pascal.npz'))
    df = {tuple(int(t) for t in k if t >= 0): float(v) for k, v in zip(g['df_keys'], g['df_vals'])}
    table = b200.rewards.CiderDTable(df, float(g['ref_len']))
    refs, cands = g['refs'].astype(np.int64), torch.from_numpy(g['cands'].astype(np.int64)).cuda()
    gts = [refs[i] for i in range(refs.shape[0])]
    scores = b200.rewards.cider_scores(gts, cands, table).cpu().numpy()
    assert np.abs(scores - g['scores']).max() < 1e-9


def _region_masks(B, R, clip):
    """Prefix masks (the collate format of dataloader.py:230-241); with ``clip`` no image uses all R regions, so clip_att shortens the axis."""
    lens = [R - 2 - (i % 3) if clip else (R if i == 0 else R - 1 - (2 * i) % (R - 2)) for i in range(B)]
    m = torch.zeros(B, R)
    for i, ln in enumerate(lens):
        m[i, :max(ln, 1)] = 1
    return m


@pytest.mark.parametrize('clip', [False, True])
@pytest.mark.parametrize('mode', ['tc_f16x3', 'simt_fp32'])
def test_scst_step_gradients_with_region_masks(mode, clip):
    """SURVEY 8(f) rank 3: variable region counts in the fused UpDown SCST step (pack_wrapper zero rows, masked-renormalised attention,
    AttModel.py:44-49,742-744) against autograd through the oracle, dropout replayed."""
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    model, fam = build_pair('updown', seed=31, logit_scale=5.0, mode=mode, **CFG)
    W = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    B, R, n, T = 5, 11, 4, CFG['T']
    fc, att = co.make_inputs(B, R, CFG['F_fc'], CFG['F_att'], seed=4)
    masks = _region_masks(B, R, clip)
    Rc = int(masks.sum(1).max())
    gts = cdo.make_refs(B, CFG['V'], seed=2)
    df, ref_len = cdo.build_document_frequency(cdo.make_refs(200, CFG['V'], seed=4))
    table = b200.rewards.CiderDTable(df, ref_len)
    model.train()
    res = model.scst_step(fc.cuda(), att.cuda(), gts, table, n, drop_prob=0.5, seed=77, att_masks=masks.cuda())
    torch.cuda.synchronize()
    sample_seq, greedy_seq = res['sample_seq'].cpu(), res['greedy_seq'].cpu()
    og, _ = co.sample(fam, fc, att, masks)
    assert torch.equal(greedy_seq, og)
    Wg = {k: v.clone().requires_grad_(True) for k, v in W.items()}
    fam_g = co.Family('updown', Wg, T)
    fam_g.drop = dropout_masks(b200, 77, 0.5, B, Rc, B * n, T, CFG['E'], CFG['H'])
    _, lp = co.sample(fam_g, fc, att, masks, sample_method='sample', sample_n=n, forced_tokens=sample_seq)
    reward, _ = cdo.self_critical_reward(greedy_seq.numpy(), gts, sample_seq.numpy(), df, ref_len)
    loss = co.reward_criterion(lp, sample_seq, torch.from_numpy(reward).float())
    loss.backward()
    assert float((res['sample_logprobs'].cpu() - lp.detach()).abs().max()) < LOGP_TOL
    assert abs(float(res['loss']) - float(loss)) < LOGP_TOL
    _check_grads(model, res['grads'], {k: v.grad for k, v in Wg.items()})


def test_xe_step_gradients_with_region_masks():
    import imagecaptioning.pytorch_b200 as b200
    model, _ = build_pair('updown', seed=31, logit_scale=5.0, mode='tc_f16x3', **CFG)
    W = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    B, R, spi, T = 4, 9, 3, CFG['T']
    fc, att = co.make_inputs(B, R, CFG['F_fc'], CFG['F_att'], seed=6)
    masks = _region_masks(B, R, True)
    Rc = int(masks.sum(1).max())
    labels, lmasks = _labels(B, spi, CFG['V'], T + 2, seed=9, short=True)
    model.train()
    res = model.xe_step(fc.cuda(), att.cuda(), labels.cuda(), lmasks.cuda(), label_smoothing=0.1, drop_prob=0.5, seed=78, att_masks=masks.cuda())
    torch.cuda.synchronize()
    Wg = {k: v.clone().requires_grad_(True) for k, v in W.items()}
    fam = co.Family('updown', Wg, T)
    fam.drop = dropout_masks(b200, 78, 0.5, B, Rc, B * spi, T + 1, CFG['E'], CFG['H'])
    lp = co.forward_teacher(fam, fc, att, labels[..., :-1], masks)
    tl, tm = labels[..., 1:].reshape(B * spi, -1), lmasks[..., 1:].reshape(B * spi, -1)
    loss = co.label_smoothing_loss(lp, tl, tm, 0.1)
    loss.backward()
    assert float((res['logprobs'].cpu() - lp.detach()).abs().max()) < LOGP_TOL
    assert abs(float(res['loss']) - float(loss)) < LOGP_TOL
    _check_grads(model, res['grads'], {k: v.grad for k, v in Wg.items()})


@pytest.mark.parametrize('clip', [False, True])
def test_aoa_scst_step_gradients_with_region_masks(clip):
    """AoANet with variable region counts: masked refiner self-attention keys, masked mean pooling (AoAModel.py:216-219) and masked decoder
    attention keys, every gradient against autograd through the oracle with all dropout masks replayed."""
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    heads = 4
    model, fam = build_pair('aoa', seed=21, logit_scale=5.0, mode='tc_f16x3', heads=heads, **AOA_CFG)
    W = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    B, R, n, T = 3, 9, 3, AOA_CFG['T']
    E, H = AOA_CFG['E'], AOA_CFG['H']
    fc, att = co.make_inputs(B, R, AOA_CFG['F_fc'], AOA_CFG['F_att'], seed=4)
    masks = _region_masks(B, R, clip)
    Rc = int(masks.sum(1).max())
    gts = cdo.make_refs(B, AOA_CFG['V'], seed=2)
    df, ref_len = cdo.build_document_frequency(cdo.make_refs(200, AOA_CFG['V'], seed=4))
    table = b200.rewards.CiderDTable(df, ref_len)
    p_lm, p_at, p_aoa, p_sub = 0.5, 0.1, 0.3, 0.1
    model.train()
    res = model.scst_step(fc.cuda(), att.cuda(), gts, table, n, drop_prob=p_lm, seed=4322, drop_attn=p_at, drop_aoa=p_aoa, drop_sublayer=p_sub, ctx_drop=1,
                          att_masks=masks.cuda())
    torch.cuda.synchronize()
    seq = res['sample_seq'].cpu()
    og, _ = co.sample(fam, fc, att, masks)
    assert torch.equal(res['greedy_seq'].cpu(), og)
    Wg = {k: v.clone().requires_grad_(True) for k, v in W.items()}
    fam_g = co.Family('aoa', Wg, T, heads=heads)
    fam_g.drop = aoa_masks(b200, 4322, B, Rc, B * n, T, E, H, heads, p_lm, p_at, p_aoa, p_sub)
    _, lp = co.sample(fam_g, fc, att, masks, sample_method='sample', sample_n=n, forced_tokens=seq)
    reward, _ = cdo.self_critical_reward(og.numpy(), gts, seq.numpy(), df, ref_len)
    loss = co.reward_criterion(lp, seq, torch.from_numpy(reward).float())
    loss.backward()
    assert float((res['sample_logprobs'].cpu() - lp.detach()).abs().max()) < LOGP_TOL
    assert abs(float(res['loss']) - float(loss)) < LOGP_TOL
    _check_grads(model, res['grads'], {k: v.grad for k, v in Wg.items()})


@pytest.mark.parametrize('family', ['updown', 'aoa'])
def test_xe_step_scheduled_sampling(family):
    """Scheduled sampling (AttModel.py:145-154) inside the fused XE step: from the second column on a row's input word is drawn from the model's
    previous prediction with probability ss_prob.  The draw cannot share torch's random stream, so the test checks (a) the hit rate, (b) that
    the draws follow exp(previous log-probs) (their mean probability against the expectation sum p^2), and (c) loss, log-probs and every
    gradient against autograd through the oracle fed with the words the engine actually used."""
    import imagecaptioning.pytorch_b200 as b200
    heads = 4
    cfg = AOA_CFG if family == 'aoa' else CFG
    model, _ = build_pair(family, seed=21, logit_scale=5.0, mode='tc_f16x3', heads=heads, **cfg)
    W = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    B, R, spi, T = 6, 9, 5, cfg['T']
    fc, att = co.make_inputs(B, R, cfg['F_fc'], cfg['F_att'], seed=4)
    labels, masks = _labels(B, spi, cfg['V'], T + 2, seed=12)
    model.train()
    model.ss_prob = 0.4
    kw = dict(drop_attn=0.0, drop_aoa=0.0, drop_sublayer=0.0, ctx_drop=1) if family == 'aoa' else {}
    res = model.xe_step(fc.cuda(), att.cuda(), labels.cuda(), masks.cuda(), label_smoothing=0.0, drop_prob=0.0, seed=991, **kw)
    torch.cuda.synchronize()
    used = res['tokens_used'].cpu()
    lab = labels[..., :-1].reshape(B * spi, -1)
    steps = int(((lab[:, 1:].sum(0) == 0).nonzero()[0]) + 1) if bool((lab[:, 1:].sum(0) == 0).any()) else lab.shape[1]
    assert torch.equal(used[:, 0], lab[:, 0])                                   # the first input is always <bos>
    cand = used[:, 1:steps] != lab[:, 1:steps]
    rate = float(cand.float().mean())
    n_cells = cand.numel()
    assert abs(rate - 0.4) < 4 * (0.4 * 0.6 / n_cells) ** 0.5 + 0.08, rate         # a draw that equals the label is not counted: slightly below 0.4
    # (c) replay in the oracle with the words that were fed
    Wg = {k: v.clone().requires_grad_(True) for k, v in W.items()}
    fam = co.Family(family, Wg, T, heads=heads)
    lp = co.forward_teacher(fam, fc, att, used.reshape(B, spi, -1))
    tl, tm = labels[..., 1:].reshape(B * spi, -1), masks[..., 1:].reshape(B * spi, -1)
    loss = co.language_model_criterion(lp, tl, tm)
    loss.backward()
    assert float((res['logprobs'].cpu() - lp.detach())[:, :steps].abs().max()) < LOGP_TOL
    assert abs(float(res['loss']) - float(loss)) < LOGP_TOL
    _check_grads(model, res['grads'], {k: v.grad for k, v in Wg.items()})
    # (b) the replaced words were drawn from exp(logprobs[:, t-1])
    p_prev = lp.detach()[:, :steps - 1].exp()
    drawn = p_prev.gather(2, used[:, 1:steps].unsqueeze(2)).squeeze(2)[cand]
    expect = (p_prev ** 2).sum(2)[cand]                                          # E[p(draw)] for a draw from p
    assert abs(float(drawn.mean()) - float(expect.mean())) < 0.15
    model.ss_prob = 0.0


@pytest.mark.parametrize('branch', ['xe', 'sc'])
def test_drop_worst_through_the_loss_wrapper(branch):
    """drop_worst_flag (tools/train.py:187-191): LossWrapper returns one loss per caption row, the trainer averages the
    k = int(rows * (1 - drop_worst_rate)) smallest and back-propagates; loss vector and every parameter gradient against autograd through
    the oracle doing literally that."""
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    model, fam = build_pair('updown', seed=31, logit_scale=5.0, mode='tc_f16x3', **CFG)
    W = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    B, R, n, spi, T = 5, 9, 4, 3, CFG['T']
    fc, att = co.make_inputs(B, R, CFG['F_fc'], CFG['F_att'], seed=5)
    labels, masks = _labels(B, spi, CFG['V'], T + 2, seed=3)
    gts = cdo.make_refs(B, CFG['V'], seed=3)
    df, ref_len = cdo.build_document_frequency(cdo.make_refs(100, CFG['V'], seed=4))
    b200.rewards.reset_scorer()
    b200.rewards.init_scorer(b200.rewards.CiderDTable(df, ref_len))
    rate = 0.3
    opt = argparse.Namespace(sc_sample_method='greedy', sc_beam_size=1, train_sample_method='sample', train_beam_size=1, train_sample_n=n,
                             cider_reward_weight=1, bleu_reward_weight=0, label_smoothing=0.0, drop_worst_rate=rate)
    lw = b200.B200LossWrapper(model, opt)
    model.train()
    model.drop_prob_lm = 0.0
    sc = branch == 'sc'
    out = lw(fc.cuda(), att.cuda(), labels.cuda(), masks.cuda(), None, gts, torch.arange(B), sc, False, True)
    rows = out['loss']
    k = int(rows.shape[0] * (1 - rate))
    assert rows.dim() == 1 and rows.shape[0] == (B * n if sc else B * spi) and rows.requires_grad
    loss = torch.topk(rows, k=k, largest=False)[0].mean()
    loss.backward()
    Wg = {k_: v.clone().requires_grad_(True) for k_, v in W.items()}
    fam_g = co.Family('updown', Wg, T)
    if sc:
        seq = lw.last_step['sample_seq'].cpu()
        greedy = lw.last_step['greedy_seq'].cpu()
        _, lp = co.sample(fam_g, fc, att, sample_method='sample', sample_n=n, forced_tokens=seq)
        reward, _ = cdo.self_critical_reward(greedy.numpy(), gts, seq.numpy(), df, ref_len)
        m = torch.cat([torch.ones(seq.shape[0], 1), (seq[:, :-1] > 0).float()], 1)
        orow = (-lp.gather(2, seq.unsqueeze(2)).squeeze(2) * torch.from_numpy(reward).float() * m).sum(1) / m.sum(1)
    else:
        lp = co.forward_teacher(fam_g, fc, att, labels[..., :-1])
        tl, tm = labels[..., 1:].reshape(B * spi, -1), masks[..., 1:].reshape(B * spi, -1)
        orow = (-lp.gather(2, tl.unsqueeze(2)).squeeze(2) * tm).sum(1) / tm.sum(1)
    oloss = torch.topk(orow, k=k, largest=False)[0].mean()
    oloss.backward()
    assert float((rows.detach().cpu() - orow.detach()).abs().max()) < LOGP_TOL
    assert abs(float(loss) - float(oloss)) < LOGP_TOL
    grads = {p: p.grad for p in model.parameters()}
    _check_grads(model, grads, {k_: v.grad for k_, v in Wg.items()})
    # any other reduction of the row vector is refused instead of silently mis-trained
    out = lw(fc.cuda(), att.cuda(), labels.cuda(), masks.cuda(), None, gts, torch.arange(B), sc, False, True)
    with pytest.raises(NotImplementedError):
        out['loss'].mean().backward()
    b200.rewards.reset_scorer()


@pytest.mark.parametrize('family', ['aoa', 'updown', 'transformer'])
def test_scst_step_graph_replay(family):
    """The SCST step is captured into a CUDA graph the second time a configuration is seen and replayed afterwards with the seed carried by
    the device-side salt (dropout.cuh).  A replay must be the same function of (weights, inputs, seed) as the eager step: the same seed
    reproduces samples, loss and gradients of the eager run; another seed draws other samples; new features / references are picked up
    (the graph reads them through the engine's staging buffers)."""
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    heads = 4
    cfg = {'aoa': AOA_CFG, 'updown': CFG, 'transformer': dict(V=40, E=32, H=64, A=2, F_fc=32, F_att=40, T=7)}[family]

    def fresh():
        m, _ = build_pair(family, seed=27, logit_scale=5.0, mode='tc_f16x3', heads=heads, **cfg)
        m.train()
        return m
    model = fresh()
    B, R, n = 3, 9, 3
    fc, att = co.make_inputs(B, R, cfg['F_fc'], cfg['F_att'], seed=4)
    fc2, att2 = co.make_inputs(B, R, cfg['F_fc'], cfg['F_att'], seed=5)
    gts = cdo.make_refs(B, cfg['V'], seed=2)
    gts2 = cdo.make_refs(B, cfg['V'], seed=3)
    df, ref_len = cdo.build_document_frequency(cdo.make_refs(200, cfg['V'], seed=4))
    table = b200.rewards.CiderDTable(df, ref_len)

    def run(m, f, a, g, seed):
        res = m.scst_step(f.cuda(), a.cuda(), g, table, n, seed=seed)
        torch.cuda.synchronize()
        return (res['sample_seq'].cpu().clone(), float(res['loss']), res['reward'].cpu().clone(), res['flat'].flat.cpu().clone(), res['greedy_seq'].cpu().clone())

    eager = run(model, fc, att, gts, 11)            # first sighting: eager (this call also binds the weights)
    l1 = model.launch_count
    other = run(model, fc, att, gts, 22)            # second: captured + launched
    l2 = model.launch_count
    replay = run(model, fc, att, gts, 11)           # third: replayed, salt = 22 ^ 11
    assert model.launch_count - l2 == l2 - l1 > 100 # the replay accounts for the launches it stands for
    assert torch.equal(replay[0], eager[0]) and torch.equal(replay[4], eager[4])
    assert abs(replay[1] - eager[1]) < 1e-6 and torch.allclose(replay[2], eager[2])
    scale = float(eager[3].abs().max())
    assert float((replay[3] - eager[3]).abs().max()) <= 1e-5 * scale          # embedding gradients use atomics: not bit-reproducible
    assert not torch.equal(other[0], eager[0])
    new_inputs = run(model, fc2, att2, gts2, 11)    # replay with other features and references
    # cross-check the replayed step on the new inputs against an engine that has never seen a graph (fresh model, eager first call)
    ref = run(fresh(), fc2, att2, gts2, 11)
    assert torch.equal(ref[0], new_inputs[0]) and abs(ref[1] - new_inputs[1]) < 1e-6
    assert float((ref[3] - new_inputs[3]).abs().max()) <= 1e-5 * float(new_inputs[3].abs().max())
