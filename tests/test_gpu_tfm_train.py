"""GPU parity of the Transformer training steps (capb200_tfm_xe_step / capb200_tfm_scst_step): loss, log-probs, reward and every parameter
gradient against torch autograd through the oracle on the CPU -- with the engine's own samples and, when dropout is on, every one of its
dropout masks replayed in the oracle -- and against what the live reference's LossWrapper + backward() produced (tests/golden/
transformer_train_small.npz, made by oracle/make_golden.py tfmtrain)."""
import argparse
import os

import numpy as np
import pytest
import torch

from helpers import LOGP_TOL, build_pair, co, tfm_masks

pytestmark = pytest.mark.gpu

# make_weights('transformer'): E = d_model, H = d_ff, A = layers per stack
CFG = dict(V=40, E=32, H=64, A=2, F_fc=32, F_att=40, T=7)
HEADS = 4


def _check_grads(model, grads, ograds, rel=5e-4):
    name_of = {id(p): k for k, p in model.state_dict(keep_vars=True).items()}
    largest = max(float(v.abs().max()) for v in ograds.values() if v is not None)
    checked = 0
    for p, g in grads.items():
        key = name_of[id(p)]
        ref = ograds[key]
        scale = float(ref.abs().max())
        err = float((g.cpu() - ref).abs().max())
        assert err <= rel * scale + 1e-7 * largest, (key, err, scale)
        checked += 1
    assert checked == sum(1 for k, v in ograds.items() if v is not None)            # every parameter (pe is a buffer)
    assert sum(float(v.abs().max()) > 1e-6 for v in ograds.values() if v is not None) >= 40


def _labels(B, spi, V, cols, seed):
    g = torch.Generator().manual_seed(seed)
    labels = torch.zeros(B, spi, cols, dtype=torch.long)
    masks = torch.zeros(B, spi, cols)
    for i in range(B):
        for j in range(spi):
            ln = int(torch.randint(1, cols - 1, (1,), generator=g))
            labels[i, j, 1:1 + ln] = torch.randint(1, V + 1, (ln,), generator=g)
            masks[i, j, :ln + 2] = 1
    return labels, masks


def _grad_weights(W):
    return {k: (v.clone().requires_grad_(True) if not k.endswith('.pe') else v.clone()) for k, v in W.items()}


@pytest.mark.parametrize('mode,dropout,smoothing,region_masks', [('tc_f16x3', False, 0.0, False), ('tc_f16x3', True, 0.1, False), ('simt_fp32', True, 0.0, True)])
def test_tfm_xe_step_gradients(mode, dropout, smoothing, region_masks):
    """Teacher-forced train-mode pass (TransformerModel.py:340-348; pad / eos keys masked, :323-328), LanguageModelCriterion / LabelSmoothing and
    every gradient against autograd through the oracle, the engine's dropout masks replayed; captions of different lengths."""
    model, _ = build_pair('transformer', seed=21, logit_scale=6.0, mode=mode, heads=HEADS, **CFG)
    W = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    B, R, spi, T = 3, 9, 2, CFG['T']
    D, Dff, layers = CFG['E'], CFG['H'], CFG['A']
    fc, att = co.make_inputs(B, R, CFG['F_fc'], CFG['F_att'], seed=4)
    labels, masks = _labels(B, spi, CFG['V'], T + 2, seed=6)
    rm = None
    if region_masks:
        rm = torch.ones(B, R)
        rm[0, 6:] = 0
        rm[2, 4:] = 0
    p_lm, p = (0.5, 0.1) if dropout else (0.0, 0.0)
    import imagecaptioning.pytorch_b200 as b200
    model.train()
    res = model.xe_step(fc.cuda(), att.cuda(), labels.cuda(), masks.cuda(), label_smoothing=smoothing, drop_prob=p_lm, dropout=p, seed=99,
                        att_masks=None if rm is None else rm.cuda())
    torch.cuda.synchronize()
    N, L = B * spi, T + 1
    Wg = _grad_weights(W)
    fam = co.Family('transformer', Wg, T, heads=HEADS)
    Rc = R if rm is None else int(rm.sum(1).max())                   # clip_att cuts the region axis to the longest valid length
    if dropout:
        fam.drop = tfm_masks(b200, 99, B, Rc, N, L, T, D, Dff, HEADS, layers, p_lm, p)
    lp = co.forward_teacher(fam, fc, att, labels[..., :-1], rm)
    flat_l, flat_m = labels.reshape(N, -1), masks.reshape(N, -1)
    loss = co.label_smoothing_loss(lp, flat_l[:, 1:], flat_m[:, 1:], smoothing) if smoothing > 0 else co.language_model_criterion(lp, flat_l[:, 1:], flat_m[:, 1:])
    loss.backward()
    assert res['logprobs'].shape == (N, L, CFG['V'] + 1)
    assert float((res['logprobs'].cpu() - lp.detach()).abs().max()) < LOGP_TOL
    assert abs(float(res['loss']) - float(loss)) < LOGP_TOL * max(1.0, abs(float(loss)))
    _check_grads(model, res['grads'], {k: (v.grad if v.requires_grad else None) for k, v in Wg.items()})


@pytest.mark.parametrize('mode,dropout,baseline', [('tc_f16x3', False, 'greedy'), ('tc_f16x3', True, 'greedy'), ('simt_fp32', True, 'leave_one_out')])
def test_tfm_scst_step_gradients(mode, dropout, baseline):
    """Self-critical step: eval-mode greedy baseline, train-mode samples drawn position by position on the K/V tape, CIDEr-D reward,
    RewardCriterion, batched backward.  Without dropout the oracle re-runs the prefix step by step like the reference's core (:351-363);
    with dropout it runs one causal pass with the engine's per-position masks."""
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    model, fam = build_pair('transformer', seed=22, logit_scale=5.0, mode=mode, heads=HEADS, **CFG)
    W = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    B, R, n, T = 3, 9, 3, CFG['T']
    D, Dff, layers = CFG['E'], CFG['H'], CFG['A']
    fc, att = co.make_inputs(B, R, CFG['F_fc'], CFG['F_att'], seed=4)
    gts = cdo.make_refs(B, CFG['V'], seed=2)
    df, ref_len = cdo.build_document_frequency(cdo.make_refs(200, CFG['V'], seed=4))
    table = b200.rewards.CiderDTable(df, ref_len)
    p_lm, p = (0.5, 0.1) if dropout else (0.0, 0.0)
    model.train()
    res = model.scst_step(fc.cuda(), att.cuda(), gts, table, n, drop_prob=p_lm, dropout=p, seed=4321, baseline=baseline)
    torch.cuda.synchronize()
    seq = res['sample_seq'].cpu()
    N = B * n
    Wg = _grad_weights(W)
    fam_g = co.Family('transformer', Wg, T, heads=HEADS)
    if dropout:
        fam_g.drop = tfm_masks(b200, 4321, B, R, N, T, T, D, Dff, HEADS, layers, p_lm, p)
        seq_in = torch.cat([torch.zeros(N, 1, dtype=torch.long), seq[:, :-1]], 1)
        lp = co.forward_teacher(fam_g, fc, att, seq_in, None, pad_keys_masked=False)
        live = torch.cat([torch.ones(N, 1, dtype=torch.bool), seq[:, :-1] > 0], 1)         # finished rows: the reference stores zero rows
        lp = lp * live.unsqueeze(2)
    else:
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
    assert float(reward.abs().max()) > 1e-3
    _check_grads(model, res['grads'], {k: (v.grad if v.requires_grad else None) for k, v in Wg.items()})


def _golden_model(golden_dir, name):
    g = np.load(os.path.join(golden_dir, name))
    cfg = dict(zip(('V', 'E', 'H', 'A', 'F_fc', 'F_att', 'T'), (int(v) for v in g['cfg'])))
    B, R, n, seed, heads, spi, _ = (int(x) for x in g['meta'])
    model, _ = build_pair('transformer', seed=seed, logit_scale=float(g['logit_scale']), mode='tc_f16x3', heads=heads, **cfg)
    fc, att = co.make_inputs(B, R, cfg['F_fc'], cfg['F_att'], seed=seed)
    return g, cfg, model, fc, att, (B, R, n, spi)


def test_tfm_training_matches_reference_golden(golden_dir):
    """Small Transformer: XE (both criteria) and SCST steps against the LIVE reference's LossWrapper + backward(), dropout 0, the reference's
    own multinomial draw replayed as forced tokens: losses, log-probs, rewards and all 93 gradient tensors."""
    import imagecaptioning.pytorch_b200 as b200
    g, cfg, model, fc, att, (B, R, n, spi) = _golden_model(golden_dir, 'transformer_train_small.npz')
    name_of = {id(p): k for k, p in model.state_dict(keep_vars=True).items()}
    labels, masks = torch.from_numpy(g['xe_labels'].astype(np.int64)), torch.from_numpy(g['xe_masks'])
    model.train()

    def check(res, prefix):
        refs = {k: g[prefix + 'g_' + k] for k in g['names']}
        largest = max(float(np.abs(v).max()) for v in refs.values())
        for p, grad in res['grads'].items():
            key = name_of[id(p)]
            ref = refs[key]
            err = float(np.abs(grad.cpu().numpy() - ref).max())
            assert err <= 5e-4 * float(np.abs(ref).max()) + 1e-7 * largest, (prefix, key, err)
        assert len(res['grads']) == len(g['names'])

    for prefix, smoothing in (('xe_', 0.0), ('xels_', 0.1)):
        res = model.xe_step(fc.cuda(), att.cuda(), labels.cuda(), masks.cuda(), label_smoothing=smoothing, drop_prob=0.0, dropout=0.0, seed=1)
        torch.cuda.synchronize()
        assert abs(float(res['loss']) - float(g[prefix + 'loss'])) < LOGP_TOL * max(1.0, abs(float(g[prefix + 'loss'])))
        if prefix == 'xe_':
            assert np.abs(res['logprobs'].cpu().numpy() - g['xe_logprobs']).max() < LOGP_TOL
        check(res, prefix)
    df = {tuple(int(t) for t in k if t >= 0): float(v) for k, v in zip(g['df_keys'], g['df_vals'])}
    table = b200.rewards.CiderDTable(df, float(g['ref_len']))
    gts = [g['gts'][i].astype(np.int64) for i in range(B)]
    forced = torch.from_numpy(g['sample_seq'].astype(np.int64))
    res = model.scst_step(fc.cuda(), att.cuda(), gts, table, n, drop_prob=0.0, dropout=0.0, seed=1, forced_tokens=forced.cuda())
    torch.cuda.synchronize()
    assert torch.equal(res['sample_seq'].cpu(), forced)
    assert np.array_equal(res['greedy_seq'].cpu().numpy(), g['greedy_seq'].astype(np.int64))
    assert np.abs(res['reward'][:, 0].double().cpu().numpy() - g['reward']).max() < LOGP_TOL
    assert abs(float(res['loss']) - float(g['sc_loss'])) < LOGP_TOL
    check(res, 'sc_')


def test_tfm_loss_wrapper_branches():
    """B200LossWrapper over the Transformer: the XE branch and the sc branch return differentiable losses whose backward() fills every
    param.grad (views of the engine's flat buffer); FusedAdam then moves every parameter."""
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    model, _ = build_pair('transformer', seed=25, logit_scale=5.0, mode='tc_f16x3', heads=HEADS, **CFG)
    B, R, n, T = 3, 9, 3, CFG['T']
    fc, att = co.make_inputs(B, R, CFG['F_fc'], CFG['F_att'], seed=4)
    labels, masks = _labels(B, 2, CFG['V'], T + 2, seed=6)
    gts = cdo.make_refs(B, CFG['V'], seed=2)
    df, ref_len = cdo.build_document_frequency(cdo.make_refs(200, CFG['V'], seed=4))
    b200.rewards.reset_scorer()
    b200.rewards.init_scorer(b200.rewards.CiderDTable(df, ref_len))
    opt = argparse.Namespace(sc_sample_method='greedy', sc_beam_size=1, train_sample_method='sample', train_beam_size=1, train_sample_n=n, cider_reward_weight=1,
                             bleu_reward_weight=0, label_smoothing=0.0)
    lw = b200.B200LossWrapper(model, opt)
    optim = b200.optim.FusedAdam(model.parameters(), lr=1e-3, clip_value=0.1)
    model.train()
    before = [p.detach().clone() for p in model.parameters()]
    for sc_flag in (False, True):
        out = lw(fc.cuda(), att.cuda(), labels.cuda(), masks.cuda(), None, gts, torch.arange(B), sc_flag, False, False)
        assert out['loss'].requires_grad and torch.isfinite(out['loss'])
        optim.zero_grad(set_to_none=True)
        out['loss'].backward()
        grads = [p.grad for p in model.parameters()]
        assert all(g_ is not None and torch.isfinite(g_).all() for g_ in grads)
        assert sum(float(g_.abs().max()) > 0 for g_ in grads) >= 80
        optim.step()
    moved = sum(float((a - b_).abs().max()) > 0 for a, b_ in zip(model.parameters(), before))
    assert moved >= 80
    b200.rewards.reset_scorer()
