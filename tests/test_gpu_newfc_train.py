"""NewFC's fused XE / SCST training steps on the H100, in both parity modes: against autograd through the restatement (newfc_oracle) with the
engine's dropout masks replayed, against the live-reference goldens of tests/make_newfc_golden.py (small and fc_rl / fc_nsc recipe size), the
step graph's replay, and B200LossWrapper with FusedAdam.  att_feats is what the reference loader hands NewFC: [B, 0, 0]."""
import argparse
import json
import os

import numpy as np
import pytest
import torch

from helpers import LOGP_TOL, PARITY_MODES, check_decode, co, family_opt
import newfc_oracle as no
from test_newfc_train_cpu import df_of, fingerprint_err

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
CFG = dict(V=40, E=32, H=48, A=24, F_fc=40, F_att=40, T=9)
GRAD_REL = 5e-4      # every gradient within 5e-4 of the tensor's largest entry


def _model(W, dims, mode):
    import imagecaptioning.pytorch_b200 as b200
    V, E, H, A, F_fc, F_att, T = dims
    m = b200.setup(family_opt('newfc', V, E, H, A, F_fc, F_att, T), numeric_mode=mode)
    m.load_state_dict(W, strict=True)
    return m.cuda().eval()


def _pair(mode, seed=31):
    W = co.make_weights('newfc', CFG['V'], CFG['E'], CFG['H'], CFG['A'], CFG['F_fc'], CFG['F_att'], seed=seed, logit_scale=5.0)
    return _model(W, tuple(CFG[k] for k in ('V', 'E', 'H', 'A', 'F_fc', 'F_att', 'T')), mode), W


def _inputs(B, seed=4):
    fc, _ = co.make_inputs(B, 1, CFG['F_fc'], CFG['F_att'], seed=seed)
    return fc, fc.new_zeros(B, 0, 0)


def _out_masks(b200, seed, p, N, steps):
    """Site 3 (core output) masks [steps, N, H], the only dropout of NewFC."""
    L, lib = b200._lib, b200._lib.load()
    out = []
    for t in range(steps):
        mm = torch.empty(N * CFG['H'], device='cuda')
        L.check(lib.capb200_dropout_mask(L.ptr(mm), N * CFG['H'], seed, 3, t, p, L.current_stream()), 'dropout_mask')
        out.append(mm.cpu().reshape(N, CFG['H']))
    return {'out': torch.stack(out)}


def _check_grads(model, grads, ograds, rel=GRAD_REL):
    name_of = {id(p): k for k, p in model.state_dict(keep_vars=True).items()}
    assert len(grads) == 9
    for p, g in grads.items():
        key = name_of[id(p)]
        ref = ograds[key]
        scale = float(ref.abs().max())
        assert scale > 0, key
        err = float((g.cpu() - ref).abs().max())
        assert err <= rel * scale + 2e-9, (key, err, scale)


def _labels(B, spi, V, L, seed):
    g = torch.Generator().manual_seed(seed)
    labels = torch.zeros(B, spi, L, dtype=torch.long)
    masks = torch.zeros(B, spi, L)
    for i in range(B):
        for j in range(spi):
            n = int(torch.randint(2, L - 1, (1,), generator=g))
            labels[i, j, 1:1 + n] = torch.randint(1, V + 1, (n,), generator=g)
            masks[i, j, :n + 2] = 1
    return labels, masks


@pytest.mark.parametrize('mode', PARITY_MODES)
@pytest.mark.parametrize('smoothing,ss_prob,keep', [(0.0, 0.0, 0), (0.1, 0.0, 0), (0.0, 0.25, 0), (0.1, 0.25, 0), (0.0, 0.0, 17)])
def test_xe_step(mode, smoothing, ss_prob, keep):
    """XE with dropout 0.5 (site 3 replayed), label smoothing, scheduled sampling (the oracle is fed the words the engine used) and
    drop_worst's keep_rows."""
    import imagecaptioning.pytorch_b200 as b200
    model, W = _pair(mode, seed=21)
    B, spi, T, p, seed = 6, 5, CFG['T'], 0.5, 991
    fc, att = _inputs(B)
    labels, masks = _labels(B, spi, CFG['V'], T + 2, seed=12)
    model.train()
    model.ss_prob = ss_prob
    res = model.xe_step(fc.cuda(), att.cuda(), labels.cuda(), masks.cuda(), label_smoothing=smoothing, drop_prob=p, seed=seed, keep_rows=keep)
    model.ss_prob = 0.0
    torch.cuda.synchronize()
    used = res['tokens_used'].cpu().reshape(B, spi, -1) if ss_prob else labels[..., :-1]
    if ss_prob:
        assert bool((used != labels[..., :-1]).any())
    Wg = {k: v.clone().requires_grad_(True) for k, v in W.items()}
    fam = no.NewFCFamily(Wg, T)
    fam.drop = _out_masks(b200, seed, p, B * spi, T + 1)
    lp = co.forward_teacher(fam, fc, att, used)
    if smoothing:
        crit = lambda red: co.label_smoothing_loss(lp, labels[..., 1:], masks[..., 1:], smoothing, reduction=red)     # noqa: E731
    else:
        crit = lambda red: co.language_model_criterion(lp, labels[..., 1:], masks[..., 1:], reduction=red)         # noqa: E731
    if keep:
        rows = crit('none')
        loss = rows.sort().values[:keep].mean()
        assert float((res['row_loss'].cpu() - rows.detach()).abs().max()) < LOGP_TOL
    else:
        loss = crit('mean')
    loss.backward()
    steps = lp.shape[1]
    assert float((res['logprobs'].cpu() - lp.detach())[:, :steps].abs().max()) < LOGP_TOL
    assert abs(float(res['loss']) - float(loss)) < LOGP_TOL
    _check_grads(model, res['grads'], {k: v.grad for k, v in Wg.items()})


@pytest.mark.parametrize('mode', PARITY_MODES)
@pytest.mark.parametrize('kind', ['greedy', 'leave_one_out', 'keep_rows'])
def test_scst_step(mode, kind):
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    model, W = _pair(mode)
    B, n, T, p, seed = 5, 4, CFG['T'], 0.5, 1234
    fc, att = _inputs(B)
    gts = cdo.make_refs(B, CFG['V'], seed=2)
    df, ref_len = cdo.build_document_frequency(cdo.make_refs(200, CFG['V'], seed=4))
    table = b200.rewards.CiderDTable(df, ref_len)
    model.train()
    keep = 13 if kind == 'keep_rows' else 0
    res = model.scst_step(fc.cuda(), att.cuda(), gts, table, n, drop_prob=p, seed=seed,
                          baseline='leave_one_out' if kind == 'leave_one_out' else 'greedy', keep_rows=keep)
    torch.cuda.synchronize()
    sseq = res['sample_seq'].cpu()
    Wg = {k: v.clone().requires_grad_(True) for k, v in W.items()}
    fam = no.NewFCFamily(Wg, T)
    if kind == 'leave_one_out':
        sc = cdo.get_scores(gts, sseq.numpy(), df, ref_len).reshape(B, n)
        reward = torch.from_numpy(np.repeat((sc - (sc.sum(1, keepdims=True) - sc) / (n - 1)).reshape(-1, 1), T, 1)).float()
    else:
        og, _ = co.sample(no.NewFCFamily(W, T), fc, att)
        assert torch.equal(res['greedy_seq'].cpu(), og)
        reward, _ = cdo.self_critical_reward(og.numpy(), gts, sseq.numpy(), df, ref_len)
        reward = torch.from_numpy(reward).float()
    fam.drop = _out_masks(b200, seed, p, B * n, T)
    _, lp = co.sample(fam, fc, att, sample_method='sample', sample_n=n, forced_tokens=sseq)
    if keep:
        rows = co.reward_criterion(lp, sseq, reward, reduction='none')
        loss = rows.sort().values[:keep].mean()
        assert float((res['row_loss'].cpu() - rows.detach()).abs().max()) < LOGP_TOL
    else:
        loss = co.reward_criterion(lp, sseq, reward)
    loss.backward()
    assert float((res['sample_logprobs'].cpu() - lp.detach()).abs().max()) < LOGP_TOL
    assert float((res['reward'].cpu() - reward).abs().max()) < LOGP_TOL
    assert abs(float(res['loss']) - float(loss)) < LOGP_TOL
    _check_grads(model, res['grads'], {k: v.grad for k, v in Wg.items()})


def test_att_masks_refused():
    """NewFC has no region features: the C ABI refuses a region mask (the Python surface ignores att_masks, as the reference does)."""
    import ctypes
    import imagecaptioning.pytorch_b200 as b200
    L, lib = b200._lib, b200._lib.load()
    model, _ = _pair('simt_fp32')
    B, spi = 2, 2
    fc, att = _inputs(B)
    labels, masks = _labels(B, spi, CFG['V'], CFG['T'] + 2, seed=1)
    model.train()
    res = model.xe_step(fc.cuda(), att.cuda(), labels.cuda(), masks.cuda(), drop_prob=0.0, att_masks=torch.ones(B, 3).cuda())
    assert torch.isfinite(res['loss'])
    fg, g = model._grad_table(lib, torch.device('cuda'))
    mk = torch.ones(B, 3, device='cuda')
    lab, msk = labels.reshape(B * spi, -1).cuda(), masks.reshape(B * spi, -1).cuda()
    lp = torch.zeros(B * spi, lab.shape[1] - 1, CFG['V'] + 1, device='cuda')
    loss = torch.empty(1, device='cuda')
    xo = L.XeOpts(spi, 3, 0, 0.0, 0.0, 1.0, L.ptr(mk), 0.0, None, 0, None)
    rc = lib.capb200_newfc_xe_step(model._engine, L.ptr(fc.cuda()), None, B, 0, ctypes.byref(xo), L.ptr(lab), L.ptr(msk), lab.shape[1], ctypes.byref(g),
                                   L.ptr(lp), L.ptr(loss), L.current_stream())
    assert rc != 0 and b'att_masks' in lib.capb200_last_error()


# ---- live-reference goldens ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('mode', PARITY_MODES)
@pytest.mark.parametrize('kind', ['xe', 'ls'])
def test_small_golden(mode, kind):
    """The reference's own draw replayed as forced tokens gives its log-probs; the XE step (LanguageModelCriterion, LabelSmoothing(0.2),
    seq_per_img 3, dropout 0) gives its loss and all 9 gradients."""
    g = np.load(os.path.join(GOLD, 'newfc_train_small.npz'))
    meta = json.loads(str(g['meta']))
    dims = tuple(int(x) for x in g['cfg'])
    V, E, H, A, F_fc, F_att, T = dims
    W = co.make_weights('newfc', V, E, H, A, F_fc, F_att, seed=meta['seed'], logit_scale=meta['logit_scale'])
    m = _model(W, dims, mode)
    B = meta['B']
    fc, _ = co.make_inputs(B, 1, F_fc, F_att, seed=meta['seed'])
    att = fc.new_zeros(B, 0, 0).cuda()
    with torch.no_grad():
        seq, lp = m(fc.cuda(), att, None, opt={'sample_n': 3}, mode='sample', forced_tokens=torch.from_numpy(g['rl_seq']).cuda())
    assert np.array_equal(seq.cpu().numpy(), g['rl_seq'])
    assert np.abs(lp.cpu().numpy() - g['rl_lp']).max() < LOGP_TOL
    m.train()
    labels, lmasks = torch.from_numpy(g['xe_labels']), torch.from_numpy(g['xe_masks'])
    res = m.xe_step(fc.cuda(), att, labels.reshape(B, 3, -1).cuda(), lmasks.reshape(B, 3, -1).cuda(), label_smoothing=0.2 if kind == 'ls' else 0.0,
                    drop_prob=0.0, seed=1)
    assert abs(float(res['loss']) - float(g[kind + '_loss'])) < LOGP_TOL
    _check_grads(m, res['grads'], {k: torch.from_numpy(g['%s_grad_%s' % (kind, k)]) for k in meta['params']})


@pytest.mark.parametrize('mode', PARITY_MODES)
@pytest.mark.parametrize('branch', ['sc', 'nsc'])
def test_recipe_size_golden(mode, branch):
    """fc_rl.yml / fc_nsc.yml sizes (10 images x 5 samples, E = H = 512, V = 9487, T = 20): the reference's LossWrapper sc and struc
    ('new_self_critical') steps replayed on their own samples match on loss, rewards and every gradient fingerprint."""
    import imagecaptioning.pytorch_b200 as b200
    g = np.load(os.path.join(GOLD, 'newfc_scst_full.npz'))
    dims = tuple(int(x) for x in g['cfg'])
    V, E, H, A, F_fc, F_att, T = dims
    B, n, seed = (int(x) for x in g['meta'])
    W = co.make_weights('newfc', V, E, H, A, F_fc, F_att, seed=seed, logit_scale=float(g['logit_scale']))
    m = _model(W, dims, mode)
    fc, _ = co.make_inputs(B, 1, F_fc, F_att, seed=seed)
    gts = [r.astype(np.int64) for r in g['gts']]
    table = b200.rewards.CiderDTable(*df_of(g))
    m.train()
    sseq = torch.from_numpy(g[branch + '_sample_seq'].astype(np.int64)).cuda()
    res = m.scst_step(fc.cuda(), fc.new_zeros(B, 0, 0).cuda(), gts, table, n, drop_prob=0.0, seed=3, forced_tokens=sseq,
                      baseline='greedy' if branch == 'sc' else 'leave_one_out')
    torch.cuda.synchronize()
    assert torch.equal(res['sample_seq'], sseq)
    if branch == 'sc':
        assert np.array_equal(res['greedy_seq'].cpu().numpy(), g['sc_greedy_seq'].astype(np.int64))
        want = g['sc_reward']
    else:
        s = g['nsc_scores'].reshape(B, n)
        want = (s - (s.sum(1, keepdims=True) - s) / (n - 1)).reshape(-1)
    assert np.abs(res['reward'][:, 0].cpu().numpy() - want).max() < LOGP_TOL
    ref_loss = float(g[branch + '_loss'])
    assert abs(float(res['loss']) - ref_loss) < LOGP_TOL * max(1.0, abs(ref_loss))
    name_of = {id(p): k for k, p in m.state_dict(keep_vars=True).items()}
    for p, grad in res['grads'].items():
        k = name_of[id(p)]
        err = fingerprint_err(grad.cpu(), g['%s_g_%s' % (branch, k)], g['%s_s_%s' % (branch, k)], g['%s_t_%s' % (branch, k)])
        assert err < GRAD_REL, (k, err)


# ---- graph replay and the training loop ------------------------------------------------------------------------------------------------

def test_step_graph_replay_identical():
    """Eager (first call), captured (second) and replayed (third) SCST steps with the same seed draw the same samples and loss."""
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    model, _ = _pair('tc_f16x3')
    B, n = 4, 3
    fc, att = _inputs(B, seed=5)
    gts = cdo.make_refs(B, CFG['V'], seed=3)
    table = b200.rewards.CiderDTable(*cdo.build_document_frequency(cdo.make_refs(100, CFG['V'], seed=4)))
    model.train()
    outs = []
    for _ in range(3):
        res = model.scst_step(fc.cuda(), att.cuda(), gts, table, n, drop_prob=0.5, seed=77)
        outs.append({'loss': res['loss'].clone(), 'seq': res['sample_seq'].clone(), 'g': [g.clone() for g in res['grads'].values()]})
    for o in outs[1:]:
        assert torch.equal(o['loss'], outs[0]['loss']) and torch.equal(o['seq'], outs[0]['seq'])
        for a, b in zip(o['g'], outs[0]['g']):          # the embedding gradient accumulates with atomics: not bit-reproducible
            assert float((a - b).abs().max()) <= 1e-5 * float(b.abs().max()) + 1e-9
    res = model.scst_step(fc.cuda(), att.cuda(), gts, table, n, drop_prob=0.5, seed=78)      # a new seed replays with new draws
    assert not torch.equal(res['sample_seq'], outs[0]['seq'])


@pytest.mark.parametrize('branch', ['xe', 'sc', 'struc'])
def test_loss_wrapper_backward_and_adam(branch):
    """fc.yml (XE with scheduled sampling), fc_rl.yml (sc) and fc_nsc.yml (struc) through B200LossWrapper, two steps with FusedAdam: param.grad
    are views of the flat gradient buffer, the weights change, and the engine decodes with the updated weights."""
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    model, _ = _pair('tc_f16x3')
    B, n = 4, 5
    fc, att = _inputs(B, seed=5)
    gts = cdo.make_refs(B, CFG['V'], seed=3)
    b200.rewards.reset_scorer()
    b200.rewards.init_scorer(b200.rewards.CiderDTable(*cdo.build_document_frequency(cdo.make_refs(100, CFG['V'], seed=4))))
    opt = argparse.Namespace(sc_sample_method='greedy', sc_beam_size=1, train_sample_method='sample', train_beam_size=1, train_sample_n=n,
                             cider_reward_weight=1, bleu_reward_weight=0, structure_loss_type='new_self_critical', structure_loss_weight=1.0,
                             label_smoothing=0.0, use_ppo=0)
    lw = b200.B200LossWrapper(model, opt)
    labels, masks = _labels(B, n, CFG['V'], CFG['T'] + 2, seed=2)
    model.train()
    model.ss_prob = 0.25 if branch == 'xe' else 0.0
    optim = b200.optim.FusedAdam(model.parameters(), lr=1e-3)
    before = {k: v.detach().clone() for k, v in model.state_dict().items()}
    try:
        for _ in range(2):
            optim.zero_grad()
            out = lw(fc.cuda(), att.cuda(), labels.cuda(), masks.cuda(), None, gts, torch.arange(B), branch == 'sc', branch == 'struc', False)
            assert out['loss'].requires_grad and torch.isfinite(out['loss'])
            out['loss'].backward()
            flat = lw.last_step['flat'].flat
            for p in model.parameters():
                assert p.grad is not None and p.grad.untyped_storage().data_ptr() == flat.untyped_storage().data_ptr()
            optim.step()                      # changes the weights: the next call re-binds them
    finally:
        model.ss_prob = 0.0
        b200.rewards.reset_scorer()
    after = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    assert all(not torch.equal(before[k].cpu(), v) for k, v in after.items())
    # the engine decodes with the updated weights: ids equal the oracle's wherever no decision is a near tie, and the engine's log-probs
    # are the updated model's (teacher-forced oracle) everywhere
    model.eval()
    with torch.no_grad():
        seq, lp = model(fc.cuda(), att.cuda(), None, opt={'beam_size': 1}, mode='sample')
    fam = no.NewFCFamily(after, CFG['T'])
    margins = []
    oseq, olp = co.sample(fam, fc, att, record_margin=margins)
    check_decode(fam, fc, att, seq, lp, oseq, olp, margins)
