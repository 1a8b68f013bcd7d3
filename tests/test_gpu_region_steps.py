"""Training steps and decoding at region counts the staged attention kernels cannot hold in shared memory, against autograd / the decoder of
the oracle on the CPU with every dropout mask replayed (DESIGN.md §2 bar: log-probs and loss within 1e-4, gradients within 5e-4 of each
tensor's largest entry):
  AoANet (H 1024, 8 heads: head width 128) XE, SCST and new_self_critical at R = 100 with prefix masks of 10..100 regions, with and without
  clipping; greedy and beam-5 decoding at R = 196; a teacher-forced backward through b200_autograd at R = 100
  Transformer XE and SCST at R = 196; SCST with 16 samples per image and 16 positions at R = 36, head width 64
  UpDown SCST with 16 samples per image at R = 300"""
import pytest
import torch

from helpers import LOGP_TOL, aoa_masks, build_pair, check_decode, co, dropout_masks, family_opt, tfm_masks
from test_gpu_scst import CFG as UD_CFG, _check_grads, _labels
from test_gpu_tfm_train import _check_grads as _tfm_check_grads, _grad_weights, _labels as _tfm_labels

pytestmark = pytest.mark.gpu

AOA = dict(V=40, E=64, H=1024, A=0, F_fc=32, F_att=48, T=7)
AOA_HEADS = 8


def _aoa_region_masks(B, R, clip):
    """Prefix masks of 10..R valid regions; with ``clip`` no image uses all R, and the longest keeps at least 76 (past the staged limit)."""
    lens = [R - 4 - 9 * i for i in range(B)] if clip else [R - (R - 10) * i // (B - 1) for i in range(B)]
    if clip:
        assert max(lens) >= 76
    m = torch.zeros(B, R)
    for i, n in enumerate(lens):
        m[i, :n] = 1
    return m


def _scst_refs(B, V):
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    gts = cdo.make_refs(B, V, seed=2)
    df, ref_len = cdo.build_document_frequency(cdo.make_refs(200, V, seed=4))
    return gts, df, ref_len, b200.rewards.CiderDTable(df, ref_len)


@pytest.mark.parametrize('clip', [False, True])
@pytest.mark.parametrize('baseline', ['greedy', 'leave_one_out'])
def test_aoa_scst_at_100_regions(baseline, clip):
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    model, fam = build_pair('aoa', seed=21, logit_scale=5.0, mode='tc_f16x3', heads=AOA_HEADS, **AOA)
    W = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    B, R, n, T = 3, 100, 2, AOA['T']
    fc, att = co.make_inputs(B, R, AOA['F_fc'], AOA['F_att'], seed=4)
    masks = _aoa_region_masks(B, R, clip)
    Rc = int(masks.sum(1).max())
    gts, df, ref_len, table = _scst_refs(B, AOA['V'])
    p_lm, p_at, p_aoa, p_sub = 0.5, 0.1, 0.3, 0.1
    model.train()
    res = model.scst_step(fc.cuda(), att.cuda(), gts, table, n, drop_prob=p_lm, seed=4323, baseline=baseline, drop_attn=p_at, drop_aoa=p_aoa,
                          drop_sublayer=p_sub, ctx_drop=1, att_masks=masks.cuda())
    torch.cuda.synchronize()
    seq = res['sample_seq'].cpu()
    Wg = {k: v.clone().requires_grad_(True) for k, v in W.items()}
    fam_g = co.Family('aoa', Wg, T, heads=AOA_HEADS)
    fam_g.drop = aoa_masks(b200, 4323, B, Rc, B * n, T, AOA['E'], AOA['H'], AOA_HEADS, p_lm, p_at, p_aoa, p_sub)
    _, lp = co.sample(fam_g, fc, att, masks, sample_method='sample', sample_n=n, forced_tokens=seq)
    if baseline == 'greedy':
        og, _ = co.sample(fam, fc, att, masks)
        assert torch.equal(res['greedy_seq'].cpu(), og)
        reward, _ = cdo.self_critical_reward(og.numpy(), gts, seq.numpy(), df, ref_len)
        loss = co.reward_criterion(lp, seq, torch.from_numpy(reward).float())
    else:
        scores = torch.from_numpy(cdo.get_scores(gts, seq.numpy(), df, ref_len))
        loss = co.new_self_critical_loss(lp, seq, scores, n)
    loss.backward()
    assert float((res['sample_logprobs'].cpu() - lp.detach()).abs().max()) < LOGP_TOL
    assert abs(float(res['loss']) - float(loss)) < LOGP_TOL
    _check_grads(model, res['grads'], {k: v.grad for k, v in Wg.items()})


@pytest.mark.parametrize('clip', [False, True])
def test_aoa_xe_at_100_regions(clip):
    import imagecaptioning.pytorch_b200 as b200
    model, _ = build_pair('aoa', seed=21, logit_scale=5.0, mode='tc_f16x3', heads=AOA_HEADS, **AOA)
    W = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    B, R, spi, T = 3, 100, 2, AOA['T']
    fc, att = co.make_inputs(B, R, AOA['F_fc'], AOA['F_att'], seed=5)
    masks = _aoa_region_masks(B, R, clip)
    Rc = int(masks.sum(1).max())
    labels, lmasks = _labels(B, spi, AOA['V'], T + 2, seed=12, short=True)
    p_lm, p_at, p_aoa, p_sub = 0.5, 0.1, 0.3, 0.1
    model.train()
    res = model.xe_step(fc.cuda(), att.cuda(), labels.cuda(), lmasks.cuda(), drop_prob=p_lm, seed=556, drop_attn=p_at, drop_aoa=p_aoa,
                        drop_sublayer=p_sub, ctx_drop=1, att_masks=masks.cuda())
    torch.cuda.synchronize()
    Wg = {k: v.clone().requires_grad_(True) for k, v in W.items()}
    fam = co.Family('aoa', Wg, T, heads=AOA_HEADS)
    fam.drop = aoa_masks(b200, 556, B, Rc, B * spi, T + 1, AOA['E'], AOA['H'], AOA_HEADS, p_lm, p_at, p_aoa, p_sub)
    lp = co.forward_teacher(fam, fc, att, labels[..., :-1], masks)
    loss = co.language_model_criterion(lp, labels[..., 1:].reshape(B * spi, -1), lmasks[..., 1:].reshape(B * spi, -1))
    loss.backward()
    assert float((res['logprobs'].cpu() - lp.detach()).abs().max()) < LOGP_TOL
    assert abs(float(res['loss']) - float(loss)) < LOGP_TOL
    _check_grads(model, res['grads'], {k: v.grad for k, v in Wg.items()})


def test_aoa_autograd_teacher_backward_at_100_regions():
    """b200_autograd = 1: model(fc, att, labels) under grad and a backward of a random upstream gradient, against oracle autograd."""
    import imagecaptioning.pytorch_b200 as b200
    W = co.make_weights('aoa', AOA['V'], AOA['E'], AOA['H'], AOA['A'], AOA['F_fc'], AOA['F_att'], seed=31, logit_scale=3.0)
    opt = family_opt('aoa', AOA['V'], AOA['E'], AOA['H'], AOA['A'], AOA['F_fc'], AOA['F_att'], AOA['T'], heads=AOA_HEADS)
    opt.b200_autograd = 1
    model = b200.setup(opt, numeric_mode='tc_f16x3')
    model.load_state_dict(W, strict=True)
    model = model.cuda().eval()
    B, R, T = 2, 100, AOA['T']
    fc, att = co.make_inputs(B, R, AOA['F_fc'], AOA['F_att'], seed=8)
    labels, _ = _labels(B, 2, AOA['V'], T + 2, seed=7)
    seq = labels[..., :-1]
    lp = model(fc.cuda(), att.cuda(), seq.cuda(), None)
    G = torch.randn(lp.shape, generator=torch.Generator().manual_seed(3))
    (lp * G.cuda()).sum().backward()
    Wg = {k: v.clone().requires_grad_(v.is_floating_point()) for k, v in W.items()}
    olp = co.forward_teacher(co.Family('aoa', Wg, T, heads=AOA_HEADS), fc, att, seq)
    assert float((lp.detach().cpu().reshape(olp.shape) - olp.detach()).abs().max()) < LOGP_TOL
    (olp * G.reshape(olp.shape)).sum().backward()
    _check_grads(model, {p: p.grad for p in model.parameters() if p.grad is not None}, {k: v.grad for k, v in Wg.items()})


@pytest.mark.parametrize('beam', [1, 5])
def test_aoa_decode_at_196_regions(beam):
    """configs/aoa.yml widths on a 14 x 14 grid: greedy and beam-5 ids bit-exact wherever the decision is not a tie."""
    cfg = dict(V=501, E=1024, H=1024, A=0, F_fc=16, F_att=2048, T=8)
    model, fam = build_pair('aoa', seed=6, logit_scale=6.0, mode='tc_f16x3', heads=8, **cfg)
    B, R = 2, 196
    fc, att = co.make_inputs(B, R, cfg['F_fc'], cfg['F_att'], seed=B + R)
    margins = []
    with torch.no_grad():
        if beam > 1:
            seq, lp = model(fc.cuda(), att.cuda(), None, opt={'beam_size': beam, 'sample_n': 1}, mode='sample')
            oseq, olp, _ = co.sample_beam(fam, fc, att, beam_size=beam, record_margin=margins)
        else:
            seq, lp = model(fc.cuda(), att.cuda(), None, opt={'sample_method': 'greedy', 'beam_size': 1, 'sample_n': 1}, mode='sample')
            oseq, olp = co.sample(fam, fc, att, record_margin=margins)
    check_decode(fam, fc, att, seq, lp, oseq, olp, margins, sample_n=1)


TFM = dict(V=40, E=32, H=64, A=2, F_fc=32, F_att=40, T=7)
TFM_HEADS = 4


def test_tfm_xe_at_196_regions():
    import imagecaptioning.pytorch_b200 as b200
    model, _ = build_pair('transformer', seed=21, logit_scale=6.0, mode='tc_f16x3', heads=TFM_HEADS, **TFM)
    W = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    B, R, spi, T = 2, 196, 2, TFM['T']
    fc, att = co.make_inputs(B, R, TFM['F_fc'], TFM['F_att'], seed=4)
    labels, masks = _tfm_labels(B, spi, TFM['V'], T + 2, seed=6)
    p_lm, p = 0.5, 0.1
    model.train()
    res = model.xe_step(fc.cuda(), att.cuda(), labels.cuda(), masks.cuda(), drop_prob=p_lm, dropout=p, seed=98)
    torch.cuda.synchronize()
    N, L = B * spi, T + 1
    Wg = _grad_weights(W)
    fam = co.Family('transformer', Wg, T, heads=TFM_HEADS)
    fam.drop = tfm_masks(b200, 98, B, R, N, L, T, TFM['E'], TFM['H'], TFM_HEADS, TFM['A'], p_lm, p)
    lp = co.forward_teacher(fam, fc, att, labels[..., :-1], None)
    flat_l, flat_m = labels.reshape(N, -1), masks.reshape(N, -1)
    loss = co.language_model_criterion(lp, flat_l[:, 1:], flat_m[:, 1:])
    loss.backward()
    assert float((res['logprobs'].cpu() - lp.detach()).abs().max()) < LOGP_TOL
    assert abs(float(res['loss']) - float(loss)) < LOGP_TOL * max(1.0, abs(float(loss)))
    _tfm_check_grads(model, res['grads'], {k: (v.grad if v.requires_grad else None) for k, v in Wg.items()})


def _tfm_scst(cfg, heads, B, R, n, seed):
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    model, fam = build_pair('transformer', seed=22, logit_scale=5.0, mode='tc_f16x3', heads=heads, **cfg)
    W = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    T = cfg['T']
    fc, att = co.make_inputs(B, R, cfg['F_fc'], cfg['F_att'], seed=4)
    gts, df, ref_len, table = _scst_refs(B, cfg['V'])
    p_lm, p = 0.5, 0.1
    model.train()
    res = model.scst_step(fc.cuda(), att.cuda(), gts, table, n, drop_prob=p_lm, dropout=p, seed=seed, baseline='greedy')
    torch.cuda.synchronize()
    seq = res['sample_seq'].cpu()
    N = B * n
    Wg = _grad_weights(W)
    fam_g = co.Family('transformer', Wg, T, heads=heads)
    fam_g.drop = tfm_masks(b200, seed, B, R, N, T, T, cfg['E'], cfg['H'], heads, cfg['A'], p_lm, p)
    seq_in = torch.cat([torch.zeros(N, 1, dtype=torch.long), seq[:, :-1]], 1)
    lp = co.forward_teacher(fam_g, fc, att, seq_in, None, pad_keys_masked=False)
    live = torch.cat([torch.ones(N, 1, dtype=torch.bool), seq[:, :-1] > 0], 1)
    lp = lp * live.unsqueeze(2)
    og, _ = co.sample(fam, fc, att)
    assert torch.equal(res['greedy_seq'].cpu(), og)
    reward, _ = cdo.self_critical_reward(og.numpy(), gts, seq.numpy(), df, ref_len)
    loss = co.reward_criterion(lp, seq, torch.from_numpy(reward).float())
    loss.backward()
    assert float((res['sample_logprobs'].cpu() - lp.detach()).abs().max()) < LOGP_TOL
    assert abs(float(res['loss']) - float(loss)) < LOGP_TOL
    _tfm_check_grads(model, res['grads'], {k: (v.grad if v.requires_grad else None) for k, v in Wg.items()})


def test_tfm_scst_at_196_regions():
    _tfm_scst(TFM, TFM_HEADS, 2, 196, 3, 4324)


def test_tfm_scst_16_samples_16_positions():
    """train_sample_n 16, seq_length 16, head width 64: the decoder attention backward runs 16 x 17 rows per image against 36 regions."""
    _tfm_scst(dict(V=40, E=128, H=64, A=2, F_fc=32, F_att=40, T=16), 2, 2, 36, 16, 4325)


def test_updown_scst_16_samples_at_300_regions():
    """The additive attention backward stages d alpha and alpha of 16 rows x 300 regions (56 KB, past the default 48 KB)."""
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    model, fam = build_pair('updown', seed=31, logit_scale=5.0, mode='tc_f16x3', **UD_CFG)
    W = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
    B, R, n, T = 2, 300, 16, UD_CFG['T']
    fc, att = co.make_inputs(B, R, UD_CFG['F_fc'], UD_CFG['F_att'], seed=4)
    gts, df, ref_len, table = _scst_refs(B, UD_CFG['V'])
    model.train()
    res = model.scst_step(fc.cuda(), att.cuda(), gts, table, n, drop_prob=0.5, seed=79)
    torch.cuda.synchronize()
    sample_seq, greedy_seq = res['sample_seq'].cpu(), res['greedy_seq'].cpu()
    og, _ = co.sample(fam, fc, att)
    assert torch.equal(greedy_seq, og)
    Wg = {k: v.clone().requires_grad_(True) for k, v in W.items()}
    fam_g = co.Family('updown', Wg, T)
    fam_g.drop = dropout_masks(b200, 79, 0.5, B, R, B * n, T, UD_CFG['E'], UD_CFG['H'])
    _, lp = co.sample(fam_g, fc, att, sample_method='sample', sample_n=n, forced_tokens=sample_seq)
    reward, _ = cdo.self_critical_reward(greedy_seq.numpy(), gts, sample_seq.numpy(), df, ref_len)
    loss = co.reward_criterion(lp, sample_seq, torch.from_numpy(reward).float())
    loss.backward()
    assert float((res['sample_logprobs'].cpu() - lp.detach()).abs().max()) < LOGP_TOL
    assert abs(float(res['loss']) - float(loss)) < LOGP_TOL
    _check_grads(model, res['grads'], {k: v.grad for k, v in Wg.items()})
