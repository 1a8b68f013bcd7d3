"""Captions past the engine's former length limits on the H100 (DESIGN.md, "Caption length"): the Transformer's decoder self-attention past
31 positions (decode, teacher forcing and every training step), CIDEr-D / BLEU-4 rewards of hypotheses and references past 64 tokens, and
beam-search records past beam x T = 1024.  EOS is suppressed (generator / logit bias of word 0 lowered by 30 in the engine and the oracle
alike), so every caption runs the full length.  Bars: DESIGN.md §2 (ids bit-exact where the decision is not a tie, log-probs and losses
within 1e-4, gradients within 5e-4 of each tensor's largest entry); float64 rewards within 1e-9 of tests/golden/long_captions.npz."""
import argparse

import numpy as np
import pytest
import torch

from helpers import LOGP_TOL, aoa_masks, check_decode, co, dropout_masks, family_opt, tfm_masks
import bleu_oracle as bo
import dbs_oracle
from test_gpu_diverse_beam import DECISIVE, P_TOL
from test_gpu_scst import _check_grads
from test_gpu_tfm_train import _check_grads as _tfm_check_grads, _grad_weights
from test_long_captions_cpu import corpus_df, load_case

pytestmark = pytest.mark.gpu

TFM = dict(V=40, E=32, H=64, A=2, F_fc=32, F_att=40)
RNN = dict(V=40, E=32, H=48, A=24, F_fc=32, F_att=40)
AOA = dict(V=40, E=32, H=64, A=0, F_fc=32, F_att=40)


def _pair(family, T, seed=5, logit_scale=5.0, mode='tc_f16x3', heads=4, V=40, E=32, H=64, A=2, F_fc=32, F_att=40):
    """(engine model, oracle Family, weights) with the bias of word 0 (EOS) lowered by 30: captions run to seq_length."""
    import imagecaptioning.pytorch_b200 as b200
    W = co.make_weights(family, V, E, H, A, F_fc, F_att, seed=seed, logit_scale=logit_scale)
    key = 'model.generator.proj.bias' if family == 'transformer' else 'logit.bias'
    W[key] = W[key].clone()
    W[key][0] -= 30.0
    model = b200.setup(family_opt(family, V, E, H, A, F_fc, F_att, T, heads), numeric_mode=mode)
    model.load_state_dict(W, strict=True)
    return model.cuda().eval(), co.Family(family, W, T, heads=heads), {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}


def _long_refs(B, V, L, seed, lo=60):
    """Five references per image of lo..L words, 0-padded to L columns."""
    rng = np.random.RandomState(seed)
    out = []
    for _ in range(B):
        rows = np.zeros((5, L), np.int64)
        for j in range(5):
            ln = rng.randint(lo, L + 1)
            rows[j, :ln] = np.minimum(rng.zipf(1.3, size=ln), V)
        out.append(rows)
    return out


def _table(V):
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    df, ref_len = cdo.build_document_frequency(cdo.make_refs(200, V, seed=4) + _long_refs(50, V, 100, seed=8))
    return df, ref_len, b200.rewards.CiderDTable(df, ref_len)


# ---- Transformer decoder self-attention: the kernels ----------------------------------------------------------------------------------

def _dec_attn(form, qkv, kc, vc, anc, labels, rows, heads, dk, t):
    import imagecaptioning.pytorch_b200 as b200
    lb, lib = b200._lib, b200._lib.load()
    D = heads * dk
    out = torch.zeros(rows, D, device='cuda')
    lb.check(lib.capb200_tfm_dec_self_attention(form, rows, heads, dk, t, lb.ptr(qkv), 3 * D, lb.ptr(kc), lb.ptr(vc), rows * D, D,
                                                lb.ptr(anc) if anc is not None else None, anc.shape[1] if anc is not None else 0,
                                                lb.ptr(labels) if labels is not None else None, labels.shape[1] if labels is not None else 0,
                                                lb.ptr(out), D, lb.current_stream()), 'tfm_dec_self_attention')
    torch.cuda.synchronize()
    return out.cpu()


def _dec_attn_f64(qkv, kc, vc, anc, labels, rows, heads, dk, t):
    D = heads * dk
    q, k, v = (x.double().reshape(rows, heads, dk) for x in qkv.cpu().split(D, 1))
    out = torch.zeros(rows, heads, dk, dtype=torch.float64)
    for r in range(rows):
        src = [int(anc[r, s]) if anc is not None else r for s in range(t)]
        K = torch.stack([kc[s, src[s]].double().reshape(heads, dk) for s in range(t)] + [k[r]], 1)       # [heads, t+1, dk]
        Vv = torch.stack([vc[s, src[s]].double().reshape(heads, dk) for s in range(t)] + [v[r]], 1)
        sc = torch.einsum('hd,hsd->hs', q[r], K) / dk ** 0.5
        if labels is not None:
            dead = torch.tensor([s > 0 and int(labels[r, s]) == 0 for s in range(t + 1)])
            sc[:, dead] = -float('inf')
        out[r] = torch.einsum('hs,hsd->hd', torch.softmax(sc, 1), Vv)
    return out.reshape(rows, D)


@pytest.mark.parametrize('dk', [8, 64, 128])
def test_dec_self_attention_forms(dk):
    """Below 32 positions the chunked kernel equals the one-lane-per-position kernel within 1e-6, and the automatic form IS the latter;
    from 32 positions on the automatic form is the chunked kernel, within 2e-5 of float64.  Beam ancestry, pad-key masking and the cache
    write of this step's k / v included."""
    torch.manual_seed(dk)
    rows, heads, T = 12, 4, 256
    D = heads * dk
    kc0, vc0 = torch.randn(T + 1, rows, D, device='cuda'), torch.randn(T + 1, rows, D, device='cuda')
    anc = torch.randint(0, rows, (rows, T), dtype=torch.int32, device='cuda')
    labels = torch.randint(0, 5, (rows, T + 1), device='cuda')
    for t in (0, 1, 17, 31, 32, 33, 100, 255, 256):
        qkv = torch.randn(rows, 3 * D, device='cuda')
        for a, lab in ((None, None), (anc, None), (anc, labels)):
            kc, vc = kc0.clone(), vc0.clone()
            got = _dec_attn(0, qkv, kc, vc, a, lab, rows, heads, dk, t)
            assert torch.equal(kc[t].cpu(), qkv[:, D:2 * D].cpu()) and torch.equal(vc[t].cpu(), qkv[:, 2 * D:].cpu())
            want = _dec_attn_f64(qkv, kc0.cpu(), vc0.cpu(), a.cpu() if a is not None else None, lab.cpu() if lab is not None else None, rows, heads,
                                 dk, t)
            assert float((got.double() - want).abs().max()) < 2e-5 * max(1.0, float(want.abs().max())), (t, a is None, lab is None)
            if t < 32:
                one_lane = _dec_attn(1, qkv, kc.clone(), vc.clone(), a, lab, rows, heads, dk, t)
                chunked = _dec_attn(2, qkv, kc.clone(), vc.clone(), a, lab, rows, heads, dk, t)
                assert torch.equal(got, one_lane)
                assert float((chunked - one_lane).abs().max()) < 1e-6, t


# ---- causal self-attention (training): staged and key-tiled ---------------------------------------------------------------------------

def _causal_f64(q, k, v, mask, heads, dk, B, T):
    def split(x):
        return x.double().reshape(B, T, heads, dk).transpose(1, 2)
    sc = torch.einsum('bhid,bhjd->bhij', split(q), split(k)) / dk ** 0.5
    allowed = torch.tril(torch.ones(T, T, dtype=torch.bool))[None, None] & (mask[:, None, None, :] != 0)
    sc = sc.masked_fill(~allowed, -float('inf'))
    return torch.einsum('bhij,bhjd->bhid', torch.softmax(sc, -1), split(v)).transpose(1, 2).reshape(B * T, heads * dk)


@pytest.mark.parametrize('T,dk', [(40, 64), (100, 64), (100, 128), (256, 128)])
def test_causal_attention_forms(T, dk):
    """The key-tiled causal forward (whole range and a one-query range, as the sampling pass calls it) and backward against float64 autograd;
    where the staged kernels fit, both forms agree, with dropout on too."""
    import imagecaptioning.pytorch_b200 as b200
    lb, lib = b200._lib, b200._lib.load()
    torch.manual_seed(T + dk)
    B, heads = 3, 2
    D = heads * dk
    q, k, v = (torch.randn(B * T, D, device='cuda') for _ in range(3))
    mask = torch.ones(B, T, device='cuda')
    mask[1, T // 2:] = 0
    mask[2, 3::7] = 0

    def fwd(form, p, q_lo=0, q_hi=T):
        out = torch.full((B * T, D), 7.0, device='cuda')
        rc = lib.capb200_mha_causal_forward(form, B, T, q_lo, q_hi, heads, dk, lb.ptr(q), lb.ptr(k), lb.ptr(v), D, lb.ptr(mask), T, 77, 50, p,
                                            lb.ptr(out), D, lb.current_stream())
        torch.cuda.synchronize()
        return rc, out.cpu()

    def bwd(form, p, d_out):
        g = [torch.zeros(B * T, D, device='cuda') for _ in range(3)]
        rc = lib.capb200_mha_causal_backward(form, B, T, heads, dk, lb.ptr(q), lb.ptr(k), lb.ptr(v), D, lb.ptr(mask), T, 77, 50, p, lb.ptr(d_out), D,
                                             lb.ptr(g[0]), lb.ptr(g[1]), lb.ptr(g[2]), D, lb.current_stream())
        torch.cuda.synchronize()
        return rc, [x.cpu() for x in g]
    qd, kd, vd = (x.cpu().double().requires_grad_(True) for x in (q, k, v))
    want = _causal_f64(qd, kd, vd, mask.cpu(), heads, dk, B, T)
    rc, tiled = fwd(2, 0.0)
    assert rc == 0 and float((tiled.double() - want.detach()).abs().max()) < 2e-5 * float(want.abs().max())
    rc, one = fwd(2, 0.0, T - 5, T - 4)
    rows = torch.arange(B) * T + T - 5
    assert rc == 0 and torch.equal(one[rows], tiled[rows]) and bool((one[torch.arange(B) * T + T - 6] == 7.0).all())
    d_out = torch.randn(B * T, D, device='cuda')
    (want * d_out.cpu().double()).sum().backward()
    rc, grads = bwd(2, 0.0, d_out)
    assert rc == 0
    for g, ref in zip(grads, (qd.grad, kd.grad, vd.grad)):
        assert float((g.double() - ref).abs().max()) < 2e-5 * float(ref.abs().max())
    for p in (0.0, 0.1):
        rc_f, staged_f = fwd(1, p)
        rc_b, staged_b = bwd(1, p, d_out)
        _, tiled_f = fwd(2, p)
        _, tiled_b = bwd(2, p, d_out)
        if rc_f == 0:
            assert float((staged_f - tiled_f).abs().max()) < 2e-5 * float(staged_f.abs().max())
        if rc_b == 0:
            for s, t_ in zip(staged_b, tiled_b):
                assert float((s - t_).abs().max()) < 2e-5 * float(s.abs().max())
    assert T * (dk + 4) * 4 * 4 + 2 * T * T * 4 <= 200 * 1024 or rc_b != 0           # the staged backward refuses where it cannot fit


# ---- Transformer decoding -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('T,beam', [(32, 1), (33, 1), (64, 1), (200, 1), (33, 3), (64, 3), (32, 5), (200, 5)])
def test_tfm_decode_long(T, beam):
    model, fam, _ = _pair('transformer', T, seed=T + beam, **TFM)
    B, R = 2, 6
    fc, att = co.make_inputs(B, R, TFM['F_fc'], TFM['F_att'], seed=T)
    masks = torch.ones(B, R)
    masks[1, 4:] = 0
    margins = []
    with torch.no_grad():
        if beam > 1:
            seq, lp = model(fc.cuda(), att.cuda(), masks.cuda(), opt={'beam_size': beam, 'sample_n': 1}, mode='sample')
            oseq, olp, _ = co.sample_beam(fam, fc, att, masks, beam_size=beam, record_margin=margins)
        else:
            seq, lp = model(fc.cuda(), att.cuda(), masks.cuda(), opt={'sample_method': 'greedy', 'beam_size': 1, 'sample_n': 1}, mode='sample')
            oseq, olp = co.sample(fam, fc, att, masks, record_margin=margins)
    assert seq.shape == (B, T) and bool((seq > 0).all())
    check_decode(fam, fc, att, seq, lp, oseq, olp, margins, masks=masks)


@pytest.mark.parametrize('T', [40, 100])
def test_tfm_teacher_forcing_long(T):
    """Teacher forcing over T + 1 positions with pad keys inside the labels masked (TransformerModel.py:324-328)."""
    model, fam, _ = _pair('transformer', T, seed=3, **TFM)
    B, spi = 2, 2
    fc, att = co.make_inputs(B, 5, TFM['F_fc'], TFM['F_att'], seed=1)
    g = torch.Generator().manual_seed(T)
    labels = torch.zeros(B, spi, T + 2, dtype=torch.long)
    for i in range(B):
        for j in range(spi):
            ln = T if i == j == 0 else int(torch.randint(T // 3, T, (1,), generator=g))
            labels[i, j, 1:1 + ln] = torch.randint(1, TFM['V'] + 1, (ln,), generator=g)
    seq = labels[..., :-1]
    with torch.no_grad():
        lp = model(fc.cuda(), att.cuda(), seq.cuda(), None)
    olp = co.forward_teacher(fam, fc, att, seq)
    assert float((lp.cpu().reshape(olp.shape) - olp).abs().max()) < LOGP_TOL


# ---- Transformer training -------------------------------------------------------------------------------------------------------

TRAIN_CASES = [(40, dict(TFM), 4), (100, dict(TFM, E=256, H=128), 2)]      # head widths 8 and 128 (the key-tiled causal backward)


@pytest.mark.parametrize('T,cfg,heads', TRAIN_CASES)
def test_tfm_xe_long(T, cfg, heads):
    import imagecaptioning.pytorch_b200 as b200
    model, _, W = _pair('transformer', T, seed=21, logit_scale=6.0, heads=heads, **cfg)
    B, R, spi = 2, 5, 2
    fc, att = co.make_inputs(B, R, cfg['F_fc'], cfg['F_att'], seed=4)
    g = torch.Generator().manual_seed(T)
    labels, masks = torch.zeros(B, spi, T + 2, dtype=torch.long), torch.zeros(B, spi, T + 2)
    for i in range(B):
        for j in range(spi):
            ln = T if i == j == 0 else int(torch.randint(T // 2, T, (1,), generator=g))
            labels[i, j, 1:1 + ln] = torch.randint(1, cfg['V'] + 1, (ln,), generator=g)
            masks[i, j, :ln + 2] = 1
    p_lm, p = 0.5, 0.1
    model.train()
    res = model.xe_step(fc.cuda(), att.cuda(), labels.cuda(), masks.cuda(), drop_prob=p_lm, dropout=p, seed=98)
    torch.cuda.synchronize()
    N, L = B * spi, T + 1
    Wg = _grad_weights(W)
    fam = co.Family('transformer', Wg, T, heads=heads)
    fam.drop = tfm_masks(b200, 98, B, R, N, L, T, cfg['E'], cfg['H'], heads, cfg['A'], p_lm, p)
    lp = co.forward_teacher(fam, fc, att, labels[..., :-1], None)
    loss = co.language_model_criterion(lp, labels.reshape(N, -1)[:, 1:], masks.reshape(N, -1)[:, 1:])
    loss.backward()
    assert float((res['logprobs'].cpu() - lp.detach()).abs().max()) < LOGP_TOL
    assert abs(float(res['loss']) - float(loss)) < LOGP_TOL * max(1.0, abs(float(loss)))
    _tfm_check_grads(model, res['grads'], {k: (v.grad if v.requires_grad else None) for k, v in Wg.items()})


@pytest.mark.parametrize('T,cfg,heads', TRAIN_CASES)
def test_tfm_new_self_critical_long(T, cfg, heads):
    """new_self_critical (leave-one-out baseline) with full-length samples: the reward scores T-token hypotheses against references of
    T - 5 .. T + 5 words (T = 100: the long CIDEr-D kernel)."""
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    model, _, W = _pair('transformer', T, seed=22, heads=heads, **cfg)
    B, R, n = 2, 5, 3
    fc, att = co.make_inputs(B, R, cfg['F_fc'], cfg['F_att'], seed=4)
    gts = _long_refs(B, cfg['V'], T + 5, seed=T, lo=T - 5)              # lengths near T: the length penalty leaves non-zero rewards
    df, ref_len, table = _table(cfg['V'])
    p_lm, p = 0.5, 0.1
    model.train()
    res = model.scst_step(fc.cuda(), att.cuda(), gts, table, n, drop_prob=p_lm, dropout=p, seed=4324, baseline='leave_one_out')
    torch.cuda.synchronize()
    seq = res['sample_seq'].cpu()
    assert bool((seq > 0).all())
    N = B * n
    Wg = _grad_weights(W)
    fam_g = co.Family('transformer', Wg, T, heads=heads)
    fam_g.drop = tfm_masks(b200, 4324, B, R, N, T, T, cfg['E'], cfg['H'], heads, cfg['A'], p_lm, p)
    seq_in = torch.cat([torch.zeros(N, 1, dtype=torch.long), seq[:, :-1]], 1)
    lp = co.forward_teacher(fam_g, fc, att, seq_in, None, pad_keys_masked=False)
    scores = torch.from_numpy(cdo.get_scores(gts, seq.numpy(), df, ref_len))
    assert float(scores.abs().max()) > 0
    loss = co.new_self_critical_loss(lp, seq, scores, n)
    loss.backward()
    assert float((res['sample_logprobs'].cpu() - lp.detach()).abs().max()) < LOGP_TOL
    assert abs(float(res['loss']) - float(loss)) < LOGP_TOL
    _tfm_check_grads(model, res['grads'], {k: (v.grad if v.requires_grad else None) for k, v in Wg.items()})


def test_tfm_scst_graph_replay_at_64():
    """The captured step graph at seq_length 64 replays the eager step: same seed, same samples, loss, reward and gradients."""
    import imagecaptioning.pytorch_b200 as b200
    model, _, _ = _pair('transformer', 64, seed=27, **TFM)
    model.train()
    B, R, n = 3, 9, 3
    fc, att = co.make_inputs(B, R, TFM['F_fc'], TFM['F_att'], seed=4)
    gts = _long_refs(B, TFM['V'], 80, seed=2)
    _, _, table = _table(TFM['V'])

    def run(seed):
        res = model.scst_step(fc.cuda(), att.cuda(), gts, table, n, seed=seed)
        torch.cuda.synchronize()
        return res['sample_seq'].cpu().clone(), float(res['loss']), res['reward'].cpu().clone(), res['flat'].flat.cpu().clone()
    eager = run(11)
    l1 = model.launch_count
    other = run(22)
    l2 = model.launch_count
    replay = run(11)
    assert model.launch_count - l2 == l2 - l1 > 100
    assert torch.equal(replay[0], eager[0]) and abs(replay[1] - eager[1]) < 1e-6 and torch.allclose(replay[2], eager[2])
    assert float((replay[3] - eager[3]).abs().max()) <= 1e-5 * float(eager[3].abs().max())
    assert not torch.equal(other[0], eager[0])


# ---- UpDown and AoANet --------------------------------------------------------------------------------------------------------------

def test_updown_scst_long():
    """UpDown self-critical step at seq_length 80 (full-length samples) against references 100 wide."""
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    T = 80
    model, fam, W = _pair('updown', T, seed=31, **RNN)
    B, R, n = 2, 7, 3
    fc, att = co.make_inputs(B, R, RNN['F_fc'], RNN['F_att'], seed=4)
    gts = _long_refs(B, RNN['V'], 100, seed=5)
    df, ref_len, table = _table(RNN['V'])
    model.train()
    res = model.scst_step(fc.cuda(), att.cuda(), gts, table, n, drop_prob=0.5, seed=79)
    torch.cuda.synchronize()
    sample_seq, greedy_seq = res['sample_seq'].cpu(), res['greedy_seq'].cpu()
    og, _ = co.sample(fam, fc, att)
    assert torch.equal(greedy_seq, og) and bool((sample_seq > 0).all())
    Wg = {k: v.clone().requires_grad_(True) for k, v in W.items()}
    fam_g = co.Family('updown', Wg, T)
    fam_g.drop = dropout_masks(b200, 79, 0.5, B, R, B * n, T, RNN['E'], RNN['H'])
    _, lp = co.sample(fam_g, fc, att, sample_method='sample', sample_n=n, forced_tokens=sample_seq)
    reward, _ = cdo.self_critical_reward(greedy_seq.numpy(), gts, sample_seq.numpy(), df, ref_len)
    assert np.abs(res['reward'].cpu().numpy() - reward).max() < 1e-5 and np.abs(reward).max() > 0
    loss = co.reward_criterion(lp, sample_seq, torch.from_numpy(reward).float())
    loss.backward()
    assert float((res['sample_logprobs'].cpu() - lp.detach()).abs().max()) < LOGP_TOL
    assert abs(float(res['loss']) - float(loss)) < LOGP_TOL
    _check_grads(model, res['grads'], {k: v.grad for k, v in Wg.items()})


@pytest.mark.parametrize('baseline', ['greedy', 'leave_one_out'])
def test_aoa_scst_long(baseline):
    """AoANet self-critical and new_self_critical steps at seq_length 80 against references 100 wide."""
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    T, heads = 80, 4
    model, fam, W = _pair('aoa', T, seed=21, heads=heads, **AOA)
    B, R, n = 2, 6, 2
    fc, att = co.make_inputs(B, R, AOA['F_fc'], AOA['F_att'], seed=4)
    gts = _long_refs(B, AOA['V'], 100, seed=6)
    df, ref_len, table = _table(AOA['V'])
    p_lm, p_at, p_aoa, p_sub = 0.5, 0.1, 0.3, 0.1
    model.train()
    res = model.scst_step(fc.cuda(), att.cuda(), gts, table, n, drop_prob=p_lm, seed=4323, baseline=baseline, drop_attn=p_at, drop_aoa=p_aoa,
                          drop_sublayer=p_sub, ctx_drop=1)
    torch.cuda.synchronize()
    seq = res['sample_seq'].cpu()
    assert bool((seq > 0).all())
    Wg = {k: v.clone().requires_grad_(True) for k, v in W.items()}
    fam_g = co.Family('aoa', Wg, T, heads=heads)
    fam_g.drop = aoa_masks(b200, 4323, B, R, B * n, T, AOA['E'], AOA['H'], heads, p_lm, p_at, p_aoa, p_sub)
    _, lp = co.sample(fam_g, fc, att, None, sample_method='sample', sample_n=n, forced_tokens=seq)
    if baseline == 'greedy':
        og, _ = co.sample(fam, fc, att)
        assert torch.equal(res['greedy_seq'].cpu(), og)
        reward, _ = cdo.self_critical_reward(og.numpy(), gts, seq.numpy(), df, ref_len)
        loss = co.reward_criterion(lp, seq, torch.from_numpy(reward).float())
    else:
        loss = co.new_self_critical_loss(lp, seq, torch.from_numpy(cdo.get_scores(gts, seq.numpy(), df, ref_len)), n)
    loss.backward()
    assert float((res['sample_logprobs'].cpu() - lp.detach()).abs().max()) < LOGP_TOL
    assert abs(float(res['loss']) - float(loss)) < LOGP_TOL
    _check_grads(model, res['grads'], {k: v.grad for k, v in Wg.items()})


def test_updown_diverse_beam_past_1024_records():
    """Diverse beam search, beam 9 in 3 groups, at seq_length 120: 3 x 120 = 360 records per group, 1080 per image."""
    T = 120
    model, fam, _ = _pair('updown', T, seed=8, **RNN)
    B, R = 4, 5
    fc, att = co.make_inputs(B, R, RNN['F_fc'], RNN['F_att'], seed=3)
    margins = []
    oseq, _, odone = dbs_oracle.diverse_sample_beam(fam, fc, att, beam_size=9, group_size=3, diversity_lambda=0.5, margin_rows=margins)
    decisive = (torch.stack(margins, 1).min(1).values > DECISIVE).numpy()
    with torch.no_grad():
        seq, lp = model(fc.cuda(), att.cuda(), None, opt={'beam_size': 9, 'group_size': 3, 'diversity_lambda': 0.5, 'sample_n': 1}, mode='sample')
    assert seq.shape == (B, T) and bool((seq > 0).all())
    assert np.array_equal(seq.cpu().numpy()[decisive], oseq.numpy()[decisive])
    for i in np.nonzero(decisive)[0]:
        for j in range(9):
            assert abs(float(model.done_beams[i][j]['p']) - float(odone[i][j]['p'])) < P_TOL * T, (i, j)
    assert decisive.sum() >= 1, decisive


# ---- standalone rewards --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('table', ['pickle', 'corpus'])
def test_rewards_against_long_golden(table):
    """CIDEr-D (capb200_cider_scores / capb200_self_critical_reward), BLEU-4 (capb200_bleu4_scores) and the weighted reward
    (capb200_weighted_reward) of 256-token rows against the reference's values: float64 within 1e-9, fp32 rewards within 1e-5."""
    import imagecaptioning.pytorch_b200 as b200
    g, gts, df, ref_len, n = load_case()
    sampled, greedy = g['sampled'], g['greedy']
    sd, gd = torch.from_numpy(sampled).cuda(), torch.from_numpy(greedy).cuda()
    pre = '' if table == 'pickle' else 'c'
    b200.rewards.reset_scorer()
    b200.rewards.init_scorer(b200.rewards.CiderDTable(df, ref_len) if table == 'pickle' else 'corpus')
    try:
        if table == 'pickle':
            bleu = b200.rewards.bleu_scores(gts, sd, greedy_res=gd).cpu().numpy()
            assert np.abs(bleu - g['bleu']).max() < 1e-9
        for j, (wc, wb) in enumerate(g['weights']):
            opt = argparse.Namespace(cider_reward_weight=float(wc), bleu_reward_weight=float(wb))
            reward = b200.rewards.get_self_critical_reward(gd, gts, sd, opt).cpu().numpy()
            assert np.abs(reward - g['%sreward_%d' % (pre, j)]).max() < 1e-5, (table, j)
            scores = b200.rewards.get_scores(gts, sd, opt).cpu().numpy()
            assert np.abs(scores - g['%sscores_%d' % (pre, j)]).max() < 1e-9, (table, j)
            cdf, clen = (df, ref_len) if table == 'pickle' else corpus_df(gts, n + 1)
            both, _ = b200.rewards.weighted_scores(gts, sd, (wc, wb), greedy_res=gd, with_reward=True)
            _, want = bo.self_critical_reward(greedy, gts, sampled, (wc, wb), cdf, clen)
            assert np.abs(both.cpu().numpy() - want).max() < 1e-9, (table, j)
        # a 65-token row against 64-token references: the long form past either bound
        short = [r[:, :64].copy() for r in gts]
        for r in short:
            r[:, 63] = 0
        opt = argparse.Namespace(cider_reward_weight=0.7, bleu_reward_weight=0.3)
        s65 = b200.rewards.get_scores(short, sd[:, :65].contiguous(), opt).cpu().numpy()
        cdf, clen = (df, ref_len) if table == 'pickle' else corpus_df(short, n)
        assert np.abs(s65 - bo.get_scores(short, sampled[:, :65], (0.7, 0.3), cdf, clen)).max() < 1e-9
    finally:
        b200.rewards.reset_scorer()


def test_rewards_refuse_past_256():
    import imagecaptioning.pytorch_b200 as b200
    g, gts, df, ref_len, n = load_case()
    b200.rewards.reset_scorer()
    b200.rewards.init_scorer(b200.rewards.CiderDTable(df, ref_len))
    try:
        wide = torch.ones(len(g['sampled']), 257, dtype=torch.long, device='cuda')
        with pytest.raises(RuntimeError, match='256'):
            b200.rewards.get_scores(gts, wide, argparse.Namespace(cider_reward_weight=1.0, bleu_reward_weight=0.0))
    finally:
        b200.rewards.reset_scorer()
