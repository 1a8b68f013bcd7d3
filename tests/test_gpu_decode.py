"""GPU parity of the whole decode path (through the Python mirror -> C ABI -> sm_90a kernels) against the oracle and the
golden vectors produced by the live reference.  Bar (BASELINE.json north_star): token ids bit-exact, log-probs within 1e-4."""
import os

import numpy as np
import pytest
import torch

from helpers import LOGP_TOL, PARITY_MODES, build_pair, check_decode, co, first_divergence

pytestmark = pytest.mark.gpu


def _golden(golden_dir, name):
    g = np.load(os.path.join(golden_dir, name))
    cfg = dict(zip(('V', 'E', 'H', 'A', 'F_fc', 'F_att', 'T'), (int(x) for x in g['cfg'])))
    B, R, b, seed = (int(x) for x in g['meta'])
    return g, cfg, B, R, b, seed


@pytest.mark.parametrize('mode', PARITY_MODES)
def test_updown_small_golden(golden_dir, mode):
    g, cfg, B, R, b, seed = _golden(golden_dir, 'updown_small.npz')
    model, fam = build_pair('updown', seed=seed, logit_scale=20.0, mode=mode, **cfg)
    fc, att = co.make_inputs(B, R, cfg['F_fc'], cfg['F_att'], seed=seed)
    fcd, attd = fc.cuda(), att.cuda()
    with torch.no_grad():
        seq, lp = model(fcd, attd, None, opt={'sample_method': 'greedy', 'beam_size': 1}, mode='sample')
        assert np.array_equal(seq.cpu().numpy(), g['greedy_seq'])
        assert np.abs(lp.cpu().numpy() - g['greedy_lp']).max() < LOGP_TOL
        seq, lp = model(fcd, attd, None, opt={'beam_size': b, 'sample_n': 1}, mode='sample')
        assert np.array_equal(seq.cpu().numpy(), g['beam_seq'])
        assert np.abs(lp.cpu().numpy() - g['beam_lp']).max() < LOGP_TOL
        for i in range(B):
            for j in range(b):
                rec = model.done_beams[i][j]
                Lr = int(g['done_len'][i, j])
                assert rec['seq'].cpu().tolist() == g['done_seq'][i, j, :Lr].tolist()
                assert abs(rec['p'] - g['done_p'][i, j]) < 1e-3
        assert tuple(model.done_beams[1][0]['logps'].shape) == (int(g['done_len'][1, 0]), cfg['V'] + 1)
        assert np.abs(model.done_beams[0][0]['logps'].cpu().numpy() - g['beam_lp'][0, :int(g['done_len'][0, 0])]).max() < LOGP_TOL
        seq, _ = model(fcd, attd, None, opt={'beam_size': b, 'sample_n': b}, mode='sample')
        assert np.array_equal(seq.cpu().numpy(), g['beamn_seq'])
        masks = torch.from_numpy(g['masks']).cuda()
        seq, lp = model(fcd, attd, masks, opt={'sample_method': 'greedy', 'beam_size': 1}, mode='sample')
        assert np.array_equal(seq.cpu().numpy(), g['masked_greedy_seq'])
        assert np.abs(lp.cpu().numpy() - g['masked_greedy_lp']).max() < LOGP_TOL
        seq, _ = model(fcd, attd, masks, opt={'beam_size': b, 'sample_n': 1}, mode='sample')
        assert np.array_equal(seq.cpu().numpy(), g['masked_beam_seq'])
        out = model(fcd, attd, torch.from_numpy(g['teacher_in']).cuda(), None)
        assert np.abs(out.cpu().numpy() - g['teacher_lp']).max() < LOGP_TOL
        forced = torch.from_numpy(g['sample_seq']).cuda()
        seq, lp = model._sample(fcd, attd, None, opt={'sample_method': 'sample', 'sample_n': 3}, forced_tokens=forced)
        assert np.array_equal(seq.cpu().numpy(), g['sample_seq'])
        assert np.abs(lp.cpu().numpy() - g['sample_lp']).max() < LOGP_TOL


@pytest.mark.parametrize('mode', PARITY_MODES)
def test_newfc_config1_golden(golden_dir, mode):
    """BASELINE.json configs[0] on the GPU: newfc greedy, batch 4, 2048-d fc feats, seq_len 16."""
    g, cfg, B, R, b, seed = _golden(golden_dir, 'newfc_cfg1.npz')
    model, fam = build_pair('newfc', seed=seed, logit_scale=12.0, mode=mode, **cfg)
    fc, att = co.make_inputs(B, 1, cfg['F_fc'], cfg['F_att'], seed=seed)
    with torch.no_grad():
        seq, lp = model(fc.cuda(), att.cuda(), None, opt={'sample_method': 'greedy', 'beam_size': 1}, mode='sample')
        picked = lp.gather(2, seq.unsqueeze(2)).squeeze(2)
        assert np.array_equal(seq.cpu().numpy(), g['greedy_seq'])
        assert np.abs(picked.cpu().numpy() - g['greedy_picked_lp']).max() < LOGP_TOL
        seq, _ = model(fc.cuda(), att.cuda(), None, opt={'beam_size': 3, 'sample_n': 1}, mode='sample')
        assert np.array_equal(seq.cpu().numpy(), g['beam_seq'])
        ps = np.array([[model.done_beams[i][j]['p'] for j in range(3)] for i in range(B)])
        assert np.abs(ps - g['done_p']).max() < 1e-3


@pytest.mark.parametrize('mode', PARITY_MODES)
def test_updown_full_dims_golden(golden_dir, mode):
    """configs/updown/updown.yml dimensions (E=H=1000, A=512, V=9487, 36 regions, T=20), beam 5 and greedy."""
    g, cfg, B, R, b, seed = _golden(golden_dir, 'updown_full.npz')
    model, fam = build_pair('updown', seed=seed, logit_scale=12.0, mode=mode, **cfg)
    fc, att = co.make_inputs(B, R, cfg['F_fc'], cfg['F_att'], seed=seed)
    with torch.no_grad():
        seq, lp = model(fc.cuda(), att.cuda(), None, opt={'sample_method': 'greedy', 'beam_size': 1}, mode='sample')
        picked = lp.gather(2, seq.unsqueeze(2)).squeeze(2)
        assert np.array_equal(seq.cpu().numpy(), g['greedy_seq']), first_divergence(seq.cpu().numpy(), g['greedy_seq'])
        assert np.abs(picked.cpu().numpy() - g['greedy_picked_lp']).max() < LOGP_TOL
        seq, lp = model(fc.cuda(), att.cuda(), None, opt={'beam_size': b, 'sample_n': 1}, mode='sample')
        assert np.array_equal(seq.cpu().numpy(), g['beam_seq']), first_divergence(seq.cpu().numpy(), g['beam_seq'])
        picked = lp.gather(2, seq.unsqueeze(2)).squeeze(2)
        assert np.abs(picked.cpu().numpy() - g['beam_picked_lp']).max() < LOGP_TOL
        ps = np.array([[model.done_beams[i][j]['p'] for j in range(b)] for i in range(B)])
        assert np.abs(ps - g['done_p']).max() < 1e-3


@pytest.mark.parametrize('mode', PARITY_MODES)
@pytest.mark.parametrize('B,R,beam', [(1, 1, 2), (9, 13, 5), (33, 36, 10), (3, 100, 1)])
def test_updown_random_shapes_vs_oracle(mode, B, R, beam):
    """Ragged / edge sizes against the oracle run live on the CPU (seeded inputs, sizes the oracle finishes in seconds)."""
    cfg = dict(V=203, E=48, H=72, A=40, F_fc=64, F_att=80, T=12)
    model, fam = build_pair('updown', seed=B * 100 + R, logit_scale=15.0, mode=mode, **cfg)
    fc, att = co.make_inputs(B, R, cfg['F_fc'], cfg['F_att'], seed=B + R)
    margins = []
    with torch.no_grad():
        if beam > 1:
            seq, lp = model(fc.cuda(), att.cuda(), None, opt={'beam_size': beam, 'sample_n': 1}, mode='sample')
            oseq, olp, odone = co.sample_beam(fam, fc, att, beam_size=beam, record_margin=margins)
        else:
            seq, lp = model(fc.cuda(), att.cuda(), None, opt={'sample_method': 'greedy', 'beam_size': 1}, mode='sample')
            oseq, olp = co.sample(fam, fc, att, record_margin=margins)
    done_p = [[model.done_beams[i][j]['p'] for j in range(beam)] for i in range(B)] if beam > 1 else None
    check_decode(fam, fc, att, seq, lp, oseq, olp, margins, done_p=done_p, odone=odone if beam > 1 else None)


def test_multinomial_sampler_distribution():
    """The sampler cannot share torch.multinomial's random stream; check it draws from softmax(logp / T): a chi-square test on
    first-step tokens over many rows of the same image, plus invariants (finished rows emit pad and zero log-prob rows)."""
    cfg = dict(V=30, E=16, H=24, A=8, F_fc=16, F_att=16, T=6)
    model, fam = build_pair('updown', seed=3, logit_scale=3.0, mode='simt_fp32', **cfg)
    fc, att = co.make_inputs(1, 4, 16, 16, seed=3)
    n = 4000
    temperature = 1.3
    torch.manual_seed(0)
    with torch.no_grad():
        seq, lp = model(fc.cuda(), att.cuda(), None, opt={'sample_method': 'sample', 'sample_n': n, 'temperature': temperature}, mode='sample')
    seq, lp = seq.cpu(), lp.cpu()
    _, olp = co.sample(fam, fc, att)
    p = torch.softmax(olp[0, 0] / temperature, 0).numpy()
    counts = np.bincount(seq[:, 0].numpy(), minlength=31).astype(np.float64)
    keep = p * n > 5
    chi2 = float((((counts - p * n) ** 2) / (p * n))[keep].sum())
    dof = int(keep.sum()) - 1
    assert chi2 < dof + 6 * (2 * dof) ** 0.5, (chi2, dof)
    assert float((lp[:, 0] - olp[0, 0]).abs().max()) < LOGP_TOL          # stored rows are the un-tempered log-probs
    ended = (seq == 0).cumsum(1) > 0
    after = torch.cat([torch.zeros(n, 1, dtype=torch.bool), ended[:, :-1]], 1)
    assert int(seq[after].abs().sum()) == 0 and float(lp[after].abs().sum()) == 0.0
    # a different seed gives a different draw; the same seed reproduces it
    torch.manual_seed(0)
    with torch.no_grad():
        seq2, _ = model(fc.cuda(), att.cuda(), None, opt={'sample_method': 'sample', 'sample_n': n, 'temperature': temperature}, mode='sample')
    assert torch.equal(seq2.cpu(), seq)


def test_scst_forward_values(golden_dir):
    """LossWrapper sc_flag branch: greedy + sampled decode + CIDEr-D reward + RewardCriterion, checked stage by stage against
    the oracle on the engine's own samples (same ids fed to the oracle)."""
    import argparse
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    cfg = dict(V=40, E=32, H=48, A=24, F_fc=32, F_att=32, T=10)
    model, fam = build_pair('updown', seed=21, logit_scale=6.0, mode='tc_f16x3', **cfg)
    model.drop_prob_lm = 0.0
    B, n = 5, 4
    fc, att = co.make_inputs(B, 9, 32, 32, seed=21)
    gts = cdo.make_refs(B, cfg['V'], seed=2)
    df, ref_len = cdo.build_document_frequency(cdo.make_refs(200, cfg['V'], seed=4))
    b200.rewards.reset_scorer()
    b200.rewards.init_scorer(b200.rewards.CiderDTable(df, ref_len))
    opt = argparse.Namespace(sc_sample_method='greedy', sc_beam_size=1, train_sample_method='sample', train_beam_size=1, train_sample_n=n,
                             cider_reward_weight=1.0, bleu_reward_weight=0.0)
    lw = b200.B200LossWrapper(model, opt)
    torch.manual_seed(1)
    out = lw(fc.cuda(), att.cuda(), None, None, None, gts, torch.arange(B), True, False, False)
    # replay on the oracle
    torch.manual_seed(1)
    model.eval()
    with torch.no_grad():
        greedy, _ = model(fc.cuda(), att.cuda(), None, opt={'sample_method': 'greedy', 'beam_size': 1}, mode='sample')
        samp, samp_lp = model(fc.cuda(), att.cuda(), None, opt={'sample_method': 'sample', 'sample_n': n}, mode='sample')
    ogreedy, _ = co.sample(fam, fc, att)
    assert torch.equal(greedy.cpu(), ogreedy)
    oseq, olp = co.sample(fam, fc, att, sample_method='sample', sample_n=n, forced_tokens=samp.cpu())
    assert float((samp_lp.cpu() - olp).abs().max()) < LOGP_TOL
    reward, _ = cdo.self_critical_reward(ogreedy.numpy(), gts, samp.cpu().numpy(), df, ref_len)
    oloss = co.reward_criterion(olp, samp.cpu(), torch.from_numpy(reward).float())
    assert abs(float(out['loss']) - float(oloss)) < LOGP_TOL
    assert abs(float(out['reward']) - float(reward[:, 0].mean())) < LOGP_TOL
    b200.rewards.reset_scorer()


@pytest.mark.parametrize('family,seed,scale', [('updown', 11, 20.0), ('transformer', 17, 10.0), ('aoa', 6, 20.0)])
def test_beam_loop_graph_replay(family, seed, scale):
    """The T-step beam loop is captured into a CUDA graph the second time a configuration is decoded and replayed afterwards: the eager
    call, the capture call and two replays (the last one on different features of the same shape) must all agree with the oracle."""
    cfg = dict(V=60, E=32, H=32, A=16, F_fc=48, F_att=48, T=8)
    if family == 'transformer':
        cfg = dict(cfg, E=32, H=64, A=2)
    model, fam = build_pair(family, seed=seed, logit_scale=scale, mode='tc_f16x3', heads=4, **cfg)
    B, R, b = 5, 7, 3
    opt = {'beam_size': b, 'sample_n': 1}
    outs = []
    with torch.no_grad():
        for call in range(4):
            fc, att = co.make_inputs(B, R, cfg['F_fc'], cfg['F_att'], seed=seed + (100 if call == 3 else 0))
            seq, lp = model(fc.cuda(), att.cuda(), None, opt=opt, mode='sample')
            outs.append((fc, att, seq.cpu().clone(), lp.cpu().clone()))
    for call in (1, 2):
        assert torch.equal(outs[call][2], outs[0][2]) and torch.equal(outs[call][3], outs[0][3])
    for fc, att, seq, lp in (outs[0], outs[3]):
        margins = []
        oseq, olp, odone = co.sample_beam(fam, fc, att, beam_size=b, record_margin=margins)
        check_decode(fam, fc, att, seq, lp, oseq, olp, margins)
    assert not torch.equal(outs[3][2], outs[0][2])


@pytest.mark.parametrize('tag,pen', [('wu', 'wu_0.5'), ('avg', 'avg_0'), ('wu2', 'wu_1.5')])
def test_beam_length_penalties_golden(golden_dir, tag, pen):
    """Beam search with opt['length_penalty'] (misc.penalty_builder) against the reference's output (tests/golden/updown_penalty.npz)."""
    g, cfg, B, R, b, seed = _golden(golden_dir, 'updown_penalty.npz')
    model, fam = build_pair('updown', seed=seed, logit_scale=20.0, mode='tc_f16x3', **cfg)
    fc, att = co.make_inputs(B, R, cfg['F_fc'], cfg['F_att'], seed=seed)
    with torch.no_grad():
        seq, lp = model(fc.cuda(), att.cuda(), None, opt={'beam_size': b, 'sample_n': 1, 'length_penalty': pen}, mode='sample')
    assert np.array_equal(seq.cpu().numpy(), g[tag + '_seq'])
    assert np.abs(lp.cpu().numpy() - g[tag + '_lp']).max() < LOGP_TOL
    for i in range(B):
        for j in range(b):
            assert abs(model.done_beams[i][j]['p'] - g[tag + '_done_p'][i, j]) < 1e-3


def test_fp16_range_guard():
    """The tensor-core decode path keeps every operand as two fp16 planes: weights or features with |x| >= 65504 (or inf / nan) must be refused, not
    silently saturated (DESIGN.md section 3).  First binding: checked synchronously.  Re-binding after an in-place weight change (what an optimizer step
    does): the conversion kernels raise a host-mapped flag and the NEXT entry point fails; capb200_range_status(1) clears it."""
    import imagecaptioning.pytorch_b200 as b200
    lib = b200._lib.load()
    cfg = dict(V=40, E=32, H=48, A=24, F_fc=32, F_att=40, T=6)
    model, _ = build_pair('updown', seed=3, logit_scale=5.0, mode='tc_f16x3', **cfg)
    fc, att = co.make_inputs(2, 5, cfg['F_fc'], cfg['F_att'], seed=1)
    opt = {'sample_method': 'greedy', 'beam_size': 1}
    with torch.no_grad():
        model.logit.weight[3, 4] = 1.0e5
        with pytest.raises(RuntimeError, match='65504'):
            model(fc.cuda(), att.cuda(), None, opt=opt, mode='sample')            # first binding: synchronous check
        assert lib.capb200_range_status(1) == 1 and lib.capb200_range_status(0) == 0
        model.logit.weight[3, 4] = 0.5
        seq, _ = model(fc.cuda(), att.cuda(), None, opt=opt, mode='sample')       # binds cleanly now
        model.logit.weight[3, 4] = float('inf')                                    # in-place change -> re-binding, not synchronised
        try:
            model(fc.cuda(), att.cuda(), None, opt=opt, mode='sample')
        except RuntimeError:
            pass
        torch.cuda.synchronize()
        with pytest.raises(RuntimeError, match='65504'):
            model(fc.cuda(), att.cuda(), None, opt=opt, mode='sample')            # the flag raised by the re-binding stops the next call
        assert lib.capb200_range_status(1) == 1
        model.logit.weight[3, 4] = 0.5
        seq2, _ = model(fc.cuda(), att.cuda(), None, opt=opt, mode='sample')
        assert torch.equal(seq, seq2)
        bad = att.clone()
        bad[0, 0, 0] = 7.0e4                                                       # features go through the same planes
        try:
            model(fc.cuda(), bad.cuda(), None, opt=opt, mode='sample')
        except RuntimeError:
            pass
        torch.cuda.synchronize()
        assert lib.capb200_range_status(1) == 1
