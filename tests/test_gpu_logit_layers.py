"""logit_layers > 1 on the H100: every decode of UpDown, Att2in2, NewFC and AoANet with AttModel's multi-layer output head (AttModel.py:87-92),
against the live-reference golden (tests/make_logit_layers_golden.py) and the oracle's head (logit_head_oracle) at k = 2 and 3, in an
ensemble, past 51 199 words and at configs[1] widths; the launch counts; and the fused XE / SCST / new_self_critical / PPO steps and the
autograd path against float64 autograd through the oracle's head with the steps' head dropout masks replayed."""
import json
import os

import numpy as np
import pytest
import torch

from helpers import LOGP_TOL, PARITY_MODES, check_decode, co, family_opt
import dbs_oracle
import ensemble_oracle as eo
import logit_head_oracle as lho

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'logit_layers_small.npz')
FAMILIES = ('updown', 'att2in2', 'newfc', 'aoa')
DECISIVE = 10 * LOGP_TOL


def _pair(fam, dims, k, seed, logit_scale, mode, heads=4):
    """(engine model on the GPU with k - 1 hidden head layers, oracle family with the same weights)"""
    import imagecaptioning.pytorch_b200 as b200
    V, E, H, A, F_fc, F_att, T = dims
    W = co.make_weights(fam, V, E, H, A, F_fc, F_att, seed=seed, logit_scale=logit_scale, logit_layers=k)
    opt = family_opt(fam, V, E, H, A, F_fc, F_att, T, heads=heads)
    opt.logit_layers = k
    m = b200.setup(opt, numeric_mode=mode)
    m.load_state_dict(W, strict=True)
    return m.cuda().eval(), (lho.family(fam, W, T, heads=heads) if k > 1 else
                             eo.member_family(fam, W, T, heads=heads)), W


def _done(model, B, beam):
    dseq = np.zeros((B, beam, model.seq_length), np.int64)
    dp = np.zeros((B, beam))
    for i in range(B):
        for j, rec in enumerate(model.done_beams[i]):
            dseq[i, j, :rec['seq'].shape[0]] = rec['seq'].cpu().numpy()
            dp[i, j] = rec['p']
    return dseq, dp


@pytest.mark.parametrize('mode', PARITY_MODES)
@pytest.mark.parametrize('fam', FAMILIES)
def test_decode_matches_reference_golden(fam, mode):
    g = np.load(GOLD)
    meta = json.loads(str(g['meta']))
    dims = tuple(int(x) for x in g['cfg'])
    m, _, _ = _pair(fam, dims, meta['logit_layers'], meta['seed'], meta['logit_scale'], mode)
    fc, att = co.make_inputs(meta['B'], meta['R'], dims[4], dims[5], seed=meta['seed'])
    p = fam + '_'
    with torch.no_grad():
        seq, lp = m(fc.cuda(), att.cuda(), None, opt={'sample_method': 'greedy', 'beam_size': 1}, mode='sample')
        assert np.array_equal(seq.cpu().numpy(), g[p + 'greedy_seq'])
        assert np.abs(lp.cpu().numpy() - g[p + 'greedy_lp']).max() < LOGP_TOL
        seq, _ = m(fc.cuda(), att.cuda(), None, opt={'beam_size': meta['beam'], 'sample_n': 1}, mode='sample')
        assert np.array_equal(seq.cpu().numpy(), g[p + 'beam_seq'])
        dseq, dp = _done(m, meta['B'], meta['beam'])
        assert np.array_equal(dseq, g[p + 'beam_done_seq'])
        assert np.abs(dp - g[p + 'beam_done_p']).max() < 1e-3
        for i in range(meta['B']):
            for j, rec in enumerate(m.done_beams[i]):
                L = rec['seq'].shape[0]
                assert np.abs(rec['logps'].cpu().numpy() - g[p + 'beam_done_logps'][i, j, :L]).max() < LOGP_TOL
        labels = torch.from_numpy(g[p + 'tf_labels'])
        lp = m(fc.cuda(), att.cuda(), labels[:, :-1].cuda(), None, mode='forward')
        assert np.abs(lp.cpu().numpy() - g[p + 'tf_lp']).max() < LOGP_TOL


@pytest.mark.parametrize('mode', PARITY_MODES)
@pytest.mark.parametrize('k', [2, 3])
@pytest.mark.parametrize('fam', FAMILIES)
def test_decode_matches_oracle(fam, k, mode):
    """Greedy, beam 3 (with done_beams), diverse beam search (families that have it), replayed samples and teacher forcing, then the same
    after an in-place change of a hidden layer's weights (the model re-binds the head)."""
    dims = (40, 32, 48, 24, 32, 40, 9)
    B, R = 4, 6
    m, fam_o, W = _pair(fam, dims, k, seed=100 + k, logit_scale=16.0, mode=mode)
    fc, att = co.make_inputs(B, R, dims[4], dims[5], seed=100 + k)
    masks = torch.ones(B, R)
    masks[1, 4:] = 0
    for rebind in (False, True):
        if rebind:
            with torch.no_grad():
                m.logit[0].weight.mul_(1.5)
                W['logit.0.weight'].mul_(1.5)
            fam_o = lho.family(fam, W, dims[-1], heads=4)
        margins = []
        oseq, olp = co.sample(fam_o, fc, att, masks, record_margin=margins)
        with torch.no_grad():
            seq, lp = m(fc.cuda(), att.cuda(), masks.cuda(), opt={'sample_method': 'greedy', 'beam_size': 1}, mode='sample')
        check_decode(fam_o, fc, att, seq, lp, oseq, olp, margins, masks=masks)
        margins = []
        oseq, olp, odone = co.sample_beam(fam_o, fc, att, masks, beam_size=3, record_margin=margins)
        with torch.no_grad():
            seq, lp = m(fc.cuda(), att.cuda(), masks.cuda(), opt={'beam_size': 3, 'sample_n': 1}, mode='sample')
        _, dp = _done(m, B, 3)
        check_decode(fam_o, fc, att, seq, lp, oseq, olp, margins, masks=masks, done_p=dp, odone=odone)
    with torch.no_grad():                        # replayed multinomial draws: the rows are the oracle's log-probs of the same prefixes
        torch.manual_seed(5)
        drawn, _ = m(fc.cuda(), att.cuda(), masks.cuda(), opt={'sample_method': 'sample', 'sample_n': 2}, mode='sample')
        seq, lp = m(fc.cuda(), att.cuda(), masks.cuda(), opt={'sample_n': 2}, mode='sample', forced_tokens=drawn)
    oseq, olp = co.sample(fam_o, fc, att, masks, sample_n=2, forced_tokens=drawn.cpu())
    assert np.array_equal(seq.cpu().numpy(), oseq.numpy())
    alive = torch.cat([torch.ones(2 * B, 1, dtype=torch.bool), (oseq[:, :-1] > 0).cumprod(1).bool()], 1)
    assert float(((lp.cpu() - olp).abs().amax(2) * alive).max()) < LOGP_TOL
    labels = torch.cat([torch.zeros(2 * B, 1, dtype=torch.long), drawn.cpu()[:, :-1]], 1)
    with torch.no_grad():
        tf = m(fc.cuda(), att.cuda(), labels.cuda(), masks.cuda(), mode='forward')
    otf = co.forward_teacher(fam_o, fc, att, labels.reshape(B, 2, -1), masks)
    assert np.abs(tf.cpu().numpy() - otf.numpy()).max() < LOGP_TOL
    if fam == 'newfc':
        return
    margins = []
    oseq, _, odone = dbs_oracle.diverse_sample_beam(fam_o, fc, att, masks, beam_size=6, group_size=3, diversity_lambda=0.5, margin_rows=margins)
    decisive = (torch.stack(margins, 1).min(1).values > DECISIVE).numpy()
    with torch.no_grad():
        seq, lp = m(fc.cuda(), att.cuda(), masks.cuda(), opt={'beam_size': 6, 'group_size': 3, 'diversity_lambda': 0.5, 'sample_n': 1}, mode='sample')
    assert decisive.any()
    assert np.array_equal(seq.cpu().numpy()[decisive], oseq.numpy()[decisive])
    dseq, dp = _done(m, B, 6)
    for i in np.nonzero(decisive)[0]:
        for j, rec in enumerate(odone[i]):
            L = rec['seq'].shape[0]
            assert np.array_equal(dseq[i, j, :L], rec['seq'].numpy())
            assert abs(dp[i, j] - float(rec['p'])) < 1e-3


@pytest.mark.parametrize('mode', PARITY_MODES)
def test_ensemble_with_a_three_layer_head_member(mode):
    """AttEnsemble of an UpDown (k = 1) and an AoANet (k = 3): greedy, beam 3 and teacher forcing against the oracle's mixture."""
    import imagecaptioning.pytorch_b200 as b200
    dims = (40, 32, 32, 16, 32, 40, 8)
    B, R = 3, 5
    m1, f1, _ = _pair('updown', dims, 1, seed=7, logit_scale=12.0, mode=mode)
    m3, f3, _ = _pair('aoa', dims, 3, seed=8, logit_scale=12.0, mode=mode)
    ens = b200.B200AttEnsemble([m1, m3], [1.0, 2.0])
    fam = eo.EnsembleFamily([f1, f3], [1.0, 2.0])
    fc, att = co.make_inputs(B, R, dims[4], dims[5], seed=9)
    with torch.no_grad():
        seq, lp = ens(fc.cuda(), att.cuda(), None, opt={'sample_method': 'greedy', 'beam_size': 1}, mode='sample')
    margins = []
    oseq, olp = co.sample(fam, fc, att, record_margin=margins)
    check_decode(fam, fc, att, seq, lp, oseq, olp, margins)
    with torch.no_grad():
        seq, lp = ens(fc.cuda(), att.cuda(), None, opt={'beam_size': 3, 'sample_n': 1}, mode='sample')
    margins = []
    oseq, olp, _ = dbs_oracle.diverse_sample_beam(fam, fc, att, beam_size=3, group_size=1, margin_rows=margins)
    decisive = (torch.stack(margins, 1).min(1).values > DECISIVE).numpy()
    assert decisive.any()
    assert np.array_equal(seq.cpu().numpy()[decisive], oseq.numpy()[decisive])
    labels = torch.cat([torch.zeros(B, 1, dtype=torch.long), oseq[:, :-1]], 1)
    with torch.no_grad():
        tf = ens(fc.cuda(), att.cuda(), labels.cuda(), None, mode='forward')
    otf = co.forward_teacher(fam, fc, att, labels.reshape(B, 1, -1))
    valid = torch.cat([torch.ones(B, 1, dtype=torch.bool), (oseq[:, :-1] > 0).cumprod(1).bool()], 1)
    assert float(((tf.cpu() - otf).abs().amax(2) * valid).max()) < LOGP_TOL


@pytest.mark.parametrize('mode', PARITY_MODES)
def test_vocabulary_above_51199_words(mode):
    """V + 1 = 52 001 (the thread-block-cluster vocabulary step) with a two-layer head: greedy and teacher forcing."""
    dims = (52000, 32, 64, 32, 32, 40, 6)
    B, R = 3, 5
    m, fam, _ = _pair('updown', dims, 2, seed=21, logit_scale=16.0, mode=mode)
    fc, att = co.make_inputs(B, R, dims[4], dims[5], seed=21)
    with torch.no_grad():
        seq, lp = m(fc.cuda(), att.cuda(), None, opt={'sample_method': 'greedy', 'beam_size': 1}, mode='sample')
    margins = []
    oseq, olp = co.sample(fam, fc, att, record_margin=margins)
    check_decode(fam, fc, att, seq, lp, oseq, olp, margins)


def test_updown_beam5_at_configs1_widths():
    """UpDown beam 5 at BASELINE configs[1]'s widths (E = H = 1000, A = 512, 2048-d features, V = 9487) with a three-layer head."""
    dims = (9487, 1000, 1000, 512, 2048, 2048, 16)
    B, R = 2, 36
    m, fam, _ = _pair('updown', dims, 3, seed=5, logit_scale=6.0, mode='tc_f16x3')
    fc, att = co.make_inputs(B, R, dims[4], dims[5], seed=5)
    with torch.no_grad():
        seq, lp = m(fc.cuda(), att.cuda(), None, opt={'beam_size': 5, 'sample_n': 1}, mode='sample')
    _, dp = _done(m, B, 5)
    margins = []
    oseq, olp, odone = co.sample_beam(fam, fc, att, beam_size=5, record_margin=margins)
    check_decode(fam, fc, att, seq, lp, oseq, olp, margins, done_p=dp, odone=odone)


@pytest.mark.parametrize('fam', FAMILIES)
def test_launch_counts(fam):
    """A decode's launches depend on k and the options only: the same for other inputs, and k - 1 more GEMMs per step than at k = 1."""
    dims = (40, 32, 48, 24, 32, 40, 9)
    B, R, T = 3, 5, dims[-1]
    counts = {}
    for k in (1, 3):
        m, _, _ = _pair(fam, dims, k, seed=3, logit_scale=12.0, mode='tc_f16x3')
        for seed in (1, 2):
            fc, att = co.make_inputs(B, R, dims[4], dims[5], seed=seed)
            for name, opt in (('greedy', {'sample_method': 'greedy', 'beam_size': 1}), ('beam', {'beam_size': 3, 'sample_n': 1})):
                with torch.no_grad():
                    m(fc.cuda(), att.cuda(), None, opt=opt, mode='sample')         # binds, sizes the workspace, sees the beam loop once
                    l0 = m.launch_count
                    m(fc.cuda(), att.cuda(), None, opt=opt, mode='sample')
                counts.setdefault((k, name), set()).add(m.launch_count - l0)
    for key, c in counts.items():
        assert len(c) == 1, (key, c)
    for name in ('greedy', 'beam'):
        (n1,), (n3,) = counts[(1, name)], counts[(3, name)]
        assert n3 - n1 == 2 * T, (name, n1, n3)      # one logit GEMM per step, NewFC's image-embedding pass included


@pytest.mark.parametrize('fam', ['updown', 'aoa'])
def test_training_needs_the_head_gradient_buffers(fam):
    """A C training entry point refuses an engine with a head whose gradient buffers were never bound, before reading anything else."""
    import imagecaptioning.pytorch_b200 as b200
    m, _, _ = _pair(fam, (40, 32, 32, 16, 32, 40, 8), 2, seed=3, logit_scale=12.0, mode='tc_f16x3')
    fc, att = co.make_inputs(2, 3, 32, 40, seed=3)
    with torch.no_grad():
        m(fc.cuda(), att.cuda(), None, opt={'beam_size': 1}, mode='sample')
    lib = b200._lib.load()
    if fam == 'updown':
        rc = lib.capb200_updown_xe_step(m._engine, None, None, 2, 3, None, None, None, 9, None, None, None, b200._lib.current_stream())
    else:
        rc = lib.capb200_aoa_xe_step(m._engine, None, 2, 3, None, None, None, 9, None, None, None, b200._lib.current_stream())
    assert rc != 0 and b'gradient buffers' in lib.capb200_last_error()


# ---- training: the fused steps and the autograd path against float64 autograd through the oracle's head, its dropout masks replayed ----
TRAIN_DIMS = (40, 32, 48, 24, 32, 40, 8)
NO_CORE_DROPOUT = {'updown': dict(drop_prob=0.0), 'att2in2': dict(drop_prob=0.0), 'newfc': dict(drop_prob=0.0),
                   'aoa': dict(drop_prob=0.0, drop_attn=0.0, drop_aoa=0.0, drop_sublayer=0.0, ctx_drop=0)}


def _labels(seed, N, T, V):
    g = torch.Generator().manual_seed(seed)
    labels = torch.zeros(N, T + 2, dtype=torch.long)
    for i in range(N):
        L = int(torch.randint(2, T + 1, (1,), generator=g))
        labels[i, 1:1 + L] = torch.randint(1, V + 1, (L,), generator=g)
    masks = torch.zeros(N, T + 2)
    for i in range(N):
        masks[i, :int((labels[i, 1:] > 0).sum()) + 2] = 1
    return labels, masks


def _head_masks(seed, k, N, steps, H, p=0.5):
    """The step's head dropout masks [k - 1][steps, N, H] (float64), regenerated from the engine's Philox streams."""
    import imagecaptioning.pytorch_b200 as b200
    L, lib = b200._lib, b200._lib.load()
    out = []
    for i in range(k - 1):
        per_t = []
        for t in range(steps):
            m = torch.empty(N * H, device='cuda')
            L.check(lib.capb200_dropout_mask(L.ptr(m), N * H, seed, lho.HEAD_DROP_SITE + i, t, p, L.current_stream()), 'dropout_mask')
            per_t.append(m.cpu().double().reshape(N, H))
        out.append(torch.stack(per_t))
    keep = float((out[0] > 0).double().mean())
    assert abs(keep - (1 - p)) < 0.05
    return out


def _oracle64(fam, W, T):
    Wg = {k: v.double().clone().requires_grad_(True) for k, v in W.items()}
    return Wg, lho.family(fam, Wg, T, heads=4)


def _check_grads(model, grads, Wg, rel=5e-4):
    name_of = {id(p): k for k, p in model.state_dict(keep_vars=True).items()}
    ograds = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in Wg.items()}
    largest = max(float(v.abs().max()) for v in ograds.values())
    names = set()
    for p, g in grads.items():
        key = name_of[id(p)]
        names.add(key)
        ref = ograds[key]
        err = float((g.detach().cpu().double() - ref).abs().max())
        assert err <= rel * float(ref.abs().max()) + 1e-7 * largest, (key, err, float(ref.abs().max()))
    assert {'logit.0.weight', 'logit.0.bias'} <= names and set(ograds) == names
    assert float(ograds['logit.0.weight'].abs().max()) > 1e-5          # the head's gradient is not vacuous


@pytest.mark.parametrize('mode', PARITY_MODES)
@pytest.mark.parametrize('fam', FAMILIES)
def test_xe_step_through_the_head(fam, mode):
    V, E, H, A, F_fc, F_att, T = TRAIN_DIMS
    B, R, spi, seed, k = 3, 5, 2, 777, 2
    m, _, W = _pair(fam, TRAIN_DIMS, k, seed=41, logit_scale=5.0, mode=mode)
    m.train()
    fc, att = co.make_inputs(B, R, F_fc, F_att, seed=41)
    labels, lmasks = _labels(5, B * spi, T, V)
    res = m.xe_step(fc.cuda(), att.cuda(), labels.cuda(), lmasks.cuda(), seed=seed, **NO_CORE_DROPOUT[fam])
    torch.cuda.synchronize()
    Wg, of = _oracle64(fam, W, T)
    of.head_drop = _head_masks(seed, k, B * spi, T + 1, H)
    lp = co.forward_teacher(of, fc.double(), att.double(), labels[:, :-1].reshape(B, spi, -1))
    loss = co.language_model_criterion(lp, labels[:, 1:], lmasks[:, 1:].double())
    loss.backward()
    assert abs(float(res['loss']) - float(loss.detach())) < LOGP_TOL
    assert float((res['logprobs'].cpu().double() - lp.detach()).abs().max()) < LOGP_TOL
    _check_grads(m, res['grads'], Wg)


@pytest.mark.parametrize('mode', PARITY_MODES)
@pytest.mark.parametrize('baseline', ['greedy', 'leave_one_out'])
@pytest.mark.parametrize('fam', FAMILIES)
def test_scst_steps_through_the_head(fam, baseline, mode):
    """The self-critical step (greedy baseline) and new_self_critical (leave-one-out): the engine's own samples and rewards, replayed with
    the head's masks; the eval-mode greedy baseline runs the head without dropout."""
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    V, E, H, A, F_fc, F_att, T = TRAIN_DIMS
    B, R, n, seed, k = 4, 5, 3, 4321, 2
    m, fam_o, W = _pair(fam, TRAIN_DIMS, k, seed=43, logit_scale=5.0, mode=mode)
    m.train()
    fc, att = co.make_inputs(B, R, F_fc, F_att, seed=43)
    gts = cdo.make_refs(B, V, seed=2)
    table = b200.rewards.CiderDTable(*cdo.build_document_frequency(cdo.make_refs(200, V, seed=4)))
    for s in (seed - 2, seed - 1, seed):        # tensor-core modes: eager, captured into a CUDA graph, replayed with the last seed
        res = m.scst_step(fc.cuda(), att.cuda(), gts, table, n, seed=s, baseline=baseline, **NO_CORE_DROPOUT[fam])
    torch.cuda.synchronize()
    seq, reward = res['sample_seq'].cpu(), res['reward'].cpu().double()
    if baseline == 'greedy':
        greedy = res['greedy_seq'].cpu()
        labels = torch.cat([torch.zeros(B, 1, dtype=torch.long), greedy[:, :-1]], 1)
        olp = co.forward_teacher(fam_o, fc, att, labels.reshape(B, 1, -1))
        top2 = olp.topk(2, dim=2).values
        alive = torch.cat([torch.ones(B, 1, dtype=torch.bool), (greedy[:, :-1] > 0).cumprod(1).bool()], 1)
        decisive = ((top2[..., 0] - top2[..., 1]) > DECISIVE) | ~alive
        assert bool((olp.argmax(2) == greedy)[decisive].all())         # the baseline is the eval-mode (no dropout) greedy decode
    Wg, of = _oracle64(fam, W, T)
    of.head_drop = _head_masks(seed, k, B * n, T, H)
    _, lp = co.sample(of, fc.double(), att.double(), sample_method='sample', sample_n=n, forced_tokens=seq)
    loss = co.reward_criterion(lp, seq, reward)
    loss.backward()
    assert float((res['sample_logprobs'].cpu().double() - lp.detach()).abs().max()) < LOGP_TOL
    assert abs(float(res['loss']) - float(loss.detach())) < LOGP_TOL
    assert float(reward.abs().max()) > 1e-3
    _check_grads(m, res['grads'], Wg)


@pytest.mark.parametrize('mode', PARITY_MODES)
def test_ppo_step_through_the_head(mode):
    """PPO on UpDown with a two-layer head: the new policy's head under dropout, the frozen old policy's (perturbed weights) in eval mode."""
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    from ppo_oracle import old_policy_input, ppo_loss
    V, E, H, A, F_fc, F_att, T = TRAIN_DIMS
    B, R, n, seed, k = 3, 5, 4, 999, 2
    m, _, W = _pair('updown', TRAIN_DIMS, k, seed=47, logit_scale=5.0, mode=mode)
    old, fam_old, W_old = _pair('updown', TRAIN_DIMS, k, seed=47, logit_scale=5.0, mode=mode)
    with torch.no_grad():
        for name, p_ in old.named_parameters():
            p_.add_(0.02 * torch.randn(p_.shape, generator=torch.Generator().manual_seed(len(name))).cuda())
            W_old[name] = p_.detach().cpu().clone()
    fam_old = lho.family('updown', W_old, T, heads=4)
    m.train()
    old.eval()
    fc, att = co.make_inputs(B, R, F_fc, F_att, seed=47)
    gts = cdo.make_refs(B, V, seed=2)
    table = b200.rewards.CiderDTable(*cdo.build_document_frequency(cdo.make_refs(200, V, seed=4)))
    res = m.ppo_step(old, fc.cuda(), att.cuda(), gts, table, n, seed=seed, drop_prob=0.0)
    torch.cuda.synchronize()
    seq = res['sample_seq'].cpu()
    Wg, of = _oracle64('updown', W, T)
    of.head_drop = _head_masks(seed, k, B * n, T, H)
    _, lp = co.sample(of, fc.double(), att.double(), sample_method='sample', sample_n=n, forced_tokens=seq)
    with torch.no_grad():
        lo = co.forward_teacher(fam_old, fc, att, old_policy_input(seq).reshape(B, n, -1)).double()
    out = ppo_loss(lp, lo, seq, res['scores'].cpu().double().reshape(-1), n)
    out['loss'].backward()
    assert abs(float(res['loss']) - float(out['loss'].detach())) < LOGP_TOL
    assert abs(float(res['kl_loss']) - float(out['kl_loss'].detach())) < LOGP_TOL
    _check_grads(m, res['grads'], Wg)


@pytest.mark.parametrize('train', [True, False])
@pytest.mark.parametrize('fam', ['updown', 'newfc'])
def test_autograd_path_through_the_head(fam, train):
    """model.autograd: differentiable teacher forcing through the head (train mode: with the head's dropout, eval mode: without)."""
    V, E, H, A, F_fc, F_att, T = TRAIN_DIMS
    B, R, spi, k = 3, 5, 2, 3
    m, _, W = _pair(fam, TRAIN_DIMS, k, seed=53, logit_scale=5.0, mode='simt_fp32')
    m.drop_prob_lm = 0.0
    m.train(train)
    m.autograd = True
    fc, att = co.make_inputs(B, R, F_fc, F_att, seed=53)
    labels, lmasks = _labels(6, B * spi, T, V)
    torch.manual_seed(11)
    seed = int(torch.randint(0, 2 ** 62, (1,)).item())
    torch.manual_seed(11)
    lp = m(fc.cuda(), att.cuda(), labels[:, :-1].cuda())
    loss = co.language_model_criterion(lp, labels[:, 1:].cuda(), lmasks[:, 1:].cuda())
    loss.backward()
    Wg, of = _oracle64(fam, W, T)
    if train:
        of.head_drop = _head_masks(seed, k, B * spi, T + 1, H)
    olp = co.forward_teacher(of, fc.double(), att.double(), labels[:, :-1].reshape(B, spi, -1))
    oloss = co.language_model_criterion(olp, labels[:, 1:], lmasks[:, 1:].double())
    oloss.backward()
    assert abs(float(loss.detach()) - float(oloss.detach())) < LOGP_TOL
    _check_grads(m, {p_: p_.grad for p_ in m.parameters()}, Wg)
