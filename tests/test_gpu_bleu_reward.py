"""The BLEU-4 reward term and the reward weights on the H100: the BLEU-4 kernel and the weighted reward against the live-reference goldens
of tests/make_bleu_golden.py, every family's fused SCST / new_self_critical step with non-default weights against autograd through the
oracles, graph replays that pick up changed weights, and the default weights' path (NULL or (1, 0)) launch for launch the CIDEr-D one."""
import argparse
import os

import numpy as np
import pytest
import torch

from helpers import LOGP_TOL, REPO, build_pair, co, family_opt
import att2in2_oracle as ao
import bleu_oracle as bo
import newfc_oracle as no
from test_bleu_reward_cpu import GOLD, full_case, syn_refs

pytestmark = pytest.mark.gpu

RNN_CFG = dict(V=40, E=32, H=48, A=24, F_fc=32, F_att=40, T=9)
AOA_CFG = dict(V=40, E=32, H=64, A=0, F_fc=32, F_att=40, T=7)
TFM_CFG = dict(V=40, E=32, H=64, A=2, F_fc=32, F_att=40, T=7)
HEADS = 4
FAMILIES = ['updown', 'att2in2', 'newfc', 'aoa', 'transformer']
GRAD_REL = 5e-4


def _family(name, mode='tc_f16x3', seed=21):
    """(engine model on the GPU in train mode, its weights on the CPU, oracle family constructor, cfg)."""
    import imagecaptioning.pytorch_b200 as b200
    cfg = {'aoa': AOA_CFG, 'transformer': TFM_CFG}.get(name, RNN_CFG)
    dims = tuple(cfg[k] for k in ('V', 'E', 'H', 'A', 'F_fc', 'F_att', 'T'))
    if name in ('att2in2', 'newfc'):
        W = co.make_weights(name, *dims[:6], seed=seed, logit_scale=5.0)
        model = b200.setup(family_opt(name, *dims), numeric_mode=mode)
        model.load_state_dict(W, strict=True)
        model = model.cuda()
        oracle = {'att2in2': lambda w: ao.Att2in2Family(w, cfg['T']), 'newfc': lambda w: no.NewFCFamily(w, cfg['T'])}[name]
    else:
        model, _ = build_pair(name, seed=seed, logit_scale=5.0, mode=mode, heads=HEADS, **cfg)
        W = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
        oracle = lambda w: co.Family(name, w, cfg['T'], heads=HEADS)      # noqa: E731
    return model.train(), W, oracle, cfg


def _inputs(name, cfg, B, seed=4):
    fc, att = co.make_inputs(B, 9, cfg['F_fc'], cfg['F_att'], seed=seed)
    if name == 'newfc':
        att = fc.new_zeros(B, 0, 0)
    return fc, att


def _scorer(cfg):
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    df, ref_len = cdo.build_document_frequency(cdo.make_refs(200, cfg['V'], seed=4))
    return df, ref_len, b200.rewards.CiderDTable(df, ref_len)


def _table_of(g):
    import imagecaptioning.pytorch_b200 as b200
    gts, sampled, greedy, df, ref_len, n = full_case(g)
    return gts, sampled, greedy, df, ref_len, n, b200.rewards.CiderDTable(df, ref_len)


# ---- kernels against the live-reference goldens -------------------------------------------------------------------------------------

def test_bleu_kernel_synthetic_golden():
    import imagecaptioning.pytorch_b200 as b200
    g = np.load(GOLD)
    hyp = torch.from_numpy(g['syn_hyp']).cuda()
    gts = [syn_refs(g, i) for i in range(hyp.shape[0])]
    got = b200.rewards.bleu_scores(gts, hyp).cpu().numpy()
    assert np.abs(got - g['syn_bleu']).max() < 1e-12


def test_bleu_kernel_pascal_golden():
    import imagecaptioning.pytorch_b200 as b200
    g = np.load(GOLD)
    z = np.load(os.path.join(REPO, 'tests', 'golden', 'ciderd_pascal.npz'))
    refs, cands = z['refs'].astype(np.int64), torch.from_numpy(z['cands'].astype(np.int64)).cuda()
    got = b200.rewards.bleu_scores([refs[i] for i in range(refs.shape[0])], cands).cpu().numpy()
    assert np.abs(got - g['pascal_bleu']).max() < 1e-12
    # with a greedy row per image appended (the layout of the self-critical reward)
    both = b200.rewards.bleu_scores([refs[i] for i in range(refs.shape[0])], cands, greedy_res=cands).cpu().numpy()
    assert np.abs(both - np.concatenate([g['pascal_bleu'], g['pascal_bleu']])).max() < 1e-12


def test_weighted_reward_golden():
    """get_self_critical_reward / get_scores with every weight pair of the golden: float64 scores within 1e-9, fp32 rewards within 1e-5;
    the leave-one-out reward of the same scores as new_self_critical computes it."""
    import imagecaptioning.pytorch_b200 as b200
    g = np.load(GOLD)
    gts, sampled, greedy, df, ref_len, n, table = _table_of(g)
    b200.rewards.reset_scorer()
    b200.rewards.init_scorer(table)
    try:
        sd, gd = torch.from_numpy(sampled).cuda(), torch.from_numpy(greedy).cuda()
        for j, (wc, wb) in enumerate(g['full_weights']):
            opt = argparse.Namespace(cider_reward_weight=float(wc), bleu_reward_weight=float(wb))
            reward = b200.rewards.get_self_critical_reward(gd, gts, sd, opt)
            assert reward.dtype == torch.float32
            assert np.abs(reward.cpu().numpy() - g['full_reward_%d' % j]).max() < 1e-5, (wc, wb)
            scores = b200.rewards.get_scores(gts, sd, opt)
            assert scores.dtype == torch.float64
            assert np.abs(scores.cpu().numpy() - g['full_scores_%d' % j]).max() < 1e-9, (wc, wb)
            both, r = b200.rewards.weighted_scores(gts, sd, (wc, wb), greedy_res=gd, with_reward=True)
            _, want = bo.self_critical_reward(greedy, gts, sampled, (wc, wb), df, ref_len)
            assert np.abs(both.cpu().numpy() - want).max() < 1e-9
            assert np.abs(r.cpu().numpy() - g['full_reward_%d' % j]).max() < 1e-5
            s, r = b200.rewards.weighted_scores(gts, sd, (wc, wb), with_reward=True)
            assert np.abs(r[:, 0].cpu().numpy() - bo.loo_reward(g['full_scores_%d' % j], n)).max() < 1e-5
            assert torch.equal(r, r[:, :1].expand_as(r))
    finally:
        b200.rewards.reset_scorer()


# ---- the fused steps -----------------------------------------------------------------------------------------------------------------

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


@pytest.mark.parametrize('family', FAMILIES)
@pytest.mark.parametrize('weights,baseline,keep', [((0.7, 0.3), 'greedy', 0), ((0.0, 1.0), 'greedy', 0), ((0.7, 0.3), 'leave_one_out', 0),
                                                   ((0.0, 1.0), 'leave_one_out', 0), ((0.7, 0.3), 'greedy', 7)])
def test_scst_step_with_weights(family, weights, baseline, keep):
    """Forced tokens (the engine's own earlier draw), dropout 0: reward and loss within 1e-4 of the restatement, every gradient against
    autograd through the family's oracle."""
    from oracle import ciderd_oracle as cdo
    model, W, oracle, cfg = _family(family)
    B, n, T = 3, 4, cfg['T']
    fc, att = _inputs(family, cfg, B)
    gts = cdo.make_refs(B, cfg['V'], seed=2)
    df, ref_len, table = _scorer(cfg)
    kw = dict(drop_prob=0.0, baseline=baseline)
    if family == 'aoa':
        kw.update(drop_attn=0.0, drop_aoa=0.0, drop_sublayer=0.0)
    if family == 'transformer':
        kw.update(dropout=0.0)
    draw = model.scst_step(fc.cuda(), att.cuda(), gts, table, n, seed=99, **kw)['sample_seq'].clone()
    gts = [r.copy() for r in gts]
    for i in range(B):                  # each image's first sample becomes a reference: 4-grams match, BLEU-4 is far from 0
        gts[i][0, :] = 0
        gts[i][0, :T] = draw[i * n].cpu().numpy()
    res = model.scst_step(fc.cuda(), att.cuda(), gts, table, n, seed=5, forced_tokens=draw, keep_rows=keep, reward_weights=weights, **kw)
    torch.cuda.synchronize()
    seq = res['sample_seq'].cpu()
    assert torch.equal(seq, draw.cpu())
    Wg = {k: (v.clone() if k.endswith('.pe') else v.clone().requires_grad_(True)) for k, v in W.items()}
    _, lp = co.sample(oracle(Wg), fc, att, sample_method='sample', sample_n=n, forced_tokens=seq)
    if baseline == 'greedy':
        og, _ = co.sample(oracle(W), fc, att)
        assert torch.equal(res['greedy_seq'].cpu(), og)
        reward, _ = bo.self_critical_reward(og.numpy(), gts, seq.numpy(), weights, df, ref_len)
        reward = torch.from_numpy(reward).float()
    else:
        scores = bo.get_scores(gts, seq.numpy(), weights, df, ref_len)
        reward = torch.from_numpy(np.repeat(bo.loo_reward(scores, n)[:, None], T, 1))
    if keep:
        rows = co.reward_criterion(lp, seq, reward, reduction='none')
        loss = rows.sort().values[:keep].mean()
        assert float((res['row_loss'].cpu() - rows.detach()).abs().max()) < LOGP_TOL
    elif baseline == 'greedy':
        loss = co.reward_criterion(lp, seq, reward)
    else:
        loss = co.new_self_critical_loss(lp, seq, torch.from_numpy(scores), n)
    loss.backward()
    assert float(reward.abs().max()) > 1e-3                       # not vacuous
    assert float((res['sample_logprobs'].cpu() - lp.detach()).abs().max()) < LOGP_TOL
    assert float((res['reward'].cpu() - reward).abs().max()) < LOGP_TOL
    assert abs(float(res['loss']) - float(loss)) < LOGP_TOL
    _check_grads(model, res['grads'], Wg)


@pytest.mark.parametrize('family', FAMILIES)
def test_graph_replay_follows_the_weights(family):
    """Eager, captured and replayed steps (no forced tokens): each call's reward is the restatement's on that call's own samples and greedy
    captions; after a change of the weights -- in the same ctypes struct contents, new values -- the next call scores with the new ones."""
    from oracle import ciderd_oracle as cdo
    model, W, oracle, cfg = _family(family)
    B, n = 3, 3
    fc, att = _inputs(family, cfg, B)
    gts = cdo.make_refs(B, cfg['V'], seed=2)
    df, ref_len, table = _scorer(cfg)
    counts = []
    for i, w in enumerate([(0.7, 0.3)] * 3 + [(0.0, 1.0)] * 3 + [(0.7, 0.3)]):
        l0 = model.launch_count
        res = model.scst_step(fc.cuda(), att.cuda(), gts, table, n, seed=100 + i, reward_weights=w)
        torch.cuda.synchronize()
        counts.append(model.launch_count - l0)
        reward, _ = bo.self_critical_reward(res['greedy_seq'].cpu().numpy(), gts, res['sample_seq'].cpu().numpy(), w, df, ref_len)
        assert np.abs(res['reward'].cpu().numpy() - reward).max() < 1e-5, (i, w)
    # the first call also binds the weights; eager, captured and replayed steps account for the same launches; (0, 1) skips the CIDEr-D kernel
    assert counts[1] == counts[2] == counts[6] and counts[3] == counts[4] == counts[5] == counts[1] - 1


@pytest.mark.parametrize('family', FAMILIES)
def test_default_weights_take_the_cider_path(family):
    """NULL and explicit (1, 0) weights issue the same launches and give bit-identical samples, log-probs, rewards and loss (the embedding
    gradient accumulates with atomics: equal to rounding); (0.7, 0.3) issues the two kernels of its extra term more."""
    from oracle import ciderd_oracle as cdo
    model, _, _, cfg = _family(family)
    B, n = 3, 3
    fc, att = _inputs(family, cfg, B)
    gts = cdo.make_refs(B, cfg['V'], seed=2)
    _, _, table = _scorer(cfg)
    draw = model.scst_step(fc.cuda(), att.cuda(), gts, table, n, seed=7)['sample_seq'].clone()
    out = {}
    for w in (None, (1.0, 0.0), (1.0, -0.5), (0.7, 0.3)):
        l0 = model.launch_count
        res = model.scst_step(fc.cuda(), att.cuda(), gts, table, n, seed=7, forced_tokens=draw, reward_weights=w)
        torch.cuda.synchronize()
        out[w] = (model.launch_count - l0, res['sample_logprobs'].clone(), res['reward'].clone(), res['loss'].clone(), res['flat'].flat.clone(),
                  res['greedy_seq'].clone())
    base = out[None]
    for w in ((1.0, 0.0), (1.0, -0.5)):
        o = out[w]
        assert o[0] == base[0]
        for a, b in zip(o[1:4] + o[5:], base[1:4] + base[5:]):
            assert torch.equal(a, b)
        assert float((o[4] - base[4]).abs().max()) <= 1e-5 * float(base[4].abs().max())
    assert out[(0.7, 0.3)][0] == base[0] + 2


@pytest.mark.parametrize('branch', ['sc', 'struc'])
def test_loss_wrapper_with_weights(branch):
    """B200LossWrapper with cider_reward_weight 0.7 and bleu_reward_weight 0.3: the fused step runs with those weights, out['reward'] of the
    struc branch is the combined fp32 score [B, n] (losses.py:61-62), that of the sc branch the mean reward of the step, and backward works."""
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    model, _, _, cfg = _family('updown')
    B, n = 3, 4
    fc, att = _inputs('updown', cfg, B)
    gts = cdo.make_refs(B, cfg['V'], seed=2)
    df, ref_len, table = _scorer(cfg)
    opt = argparse.Namespace(sc_sample_method='greedy', sc_beam_size=1, train_sample_method='sample', train_beam_size=1, train_sample_n=n,
                             cider_reward_weight=0.7, bleu_reward_weight=0.3, structure_loss_type='new_self_critical', structure_loss_weight=1.0,
                             label_smoothing=0.0, use_ppo=0)
    b200.rewards.reset_scorer()
    b200.rewards.init_scorer(table)
    try:
        lw = b200.B200LossWrapper(model, opt)
        labels = torch.zeros(B, n, cfg['T'] + 2, dtype=torch.long)
        out = lw(fc.cuda(), att.cuda(), labels.cuda(), torch.ones_like(labels, dtype=torch.float32).cuda(), None, gts, torch.arange(B),
                 branch == 'sc', branch == 'struc', False)
        out['loss'].backward()
        torch.cuda.synchronize()
        seq = lw.last_step['sample_seq'].cpu().numpy()
        if branch == 'struc':
            want = bo.get_scores(gts, seq, (0.7, 0.3), df, ref_len).astype(np.float32).reshape(B, n)
            assert out['reward'].shape == (B, n) and np.abs(out['reward'].cpu().numpy() - want).max() < 1e-5
        else:
            reward, _ = bo.self_critical_reward(lw.last_step['greedy_seq'].cpu().numpy(), gts, seq, (0.7, 0.3), df, ref_len)
            assert abs(float(out['reward']) - float(reward[:, 0].astype(np.float32).mean())) < 1e-5
        assert all(p.grad is not None for p in model.parameters())
    finally:
        b200.rewards.reset_scorer()
