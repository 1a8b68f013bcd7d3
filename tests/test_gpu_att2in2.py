"""Att2in2 on the H100: decoding against the live-reference goldens (tests/make_att2in2_golden.py) and the fused XE / SCST steps against
autograd through the restatement (att2in2_oracle), in both parity modes."""
import argparse
import json
import os

import numpy as np
import pytest
import torch

from helpers import LOGP_TOL, PARITY_MODES, att2in2_masks, co, family_opt
import att2in2_oracle as ao
import dbs_oracle

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
CFG = dict(V=40, E=32, H=48, A=24, F_fc=32, F_att=40, T=9)


def _model(W, dims, mode):
    import imagecaptioning.pytorch_b200 as b200
    V, E, H, A, F_fc, F_att, T = dims
    m = b200.setup(family_opt('att2in2', V, E, H, A, F_fc, F_att, T), numeric_mode=mode)
    m.load_state_dict(W, strict=True)
    return m.cuda().eval()


def _small(mode):
    g = np.load(os.path.join(GOLD, 'att2in2_small.npz'))
    meta = json.loads(str(g['meta']))
    dims = tuple(int(x) for x in g['cfg'])
    V, E, H, A, F_fc, F_att, T = dims
    W = co.make_weights('att2in2', V, E, H, A, F_fc, F_att, seed=meta['seed'], logit_scale=meta['logit_scale'])
    fc, att = co.make_inputs(meta['B'], meta['R'], F_fc, F_att, seed=meta['seed'])
    masks = torch.ones(meta['B'], meta['R'])
    masks[1, 5:] = 0
    masks[3, 3:] = 0
    return g, _model(W, dims, mode), ao.Att2in2Family(W, T), fc, att, masks, T


@pytest.mark.parametrize('mode', PARITY_MODES)
def test_decode_goldens(mode):
    g, m, fam, fc, att, masks, T = _small(mode)
    with torch.no_grad():
        for tag, mk in (('', None), ('masked_', masks)):
            seq, lp = m(fc.cuda(), att.cuda(), None if mk is None else mk.cuda(), opt={'beam_size': 1}, mode='sample')
            assert np.array_equal(seq.cpu().numpy(), g[tag + 'greedy_seq'])
            assert np.abs(lp.cpu().numpy() - g[tag + 'greedy_lp']).max() < LOGP_TOL
        seq, lp = m(fc.cuda(), att.cuda(), None, opt={'sample_n': 3}, mode='sample', forced_tokens=torch.from_numpy(g['sample_seq']).cuda())
        assert np.array_equal(seq.cpu().numpy(), g['sample_seq'])
        assert np.abs(lp.cpu().numpy() - g['sample_lp']).max() < LOGP_TOL
        labels = torch.from_numpy(g['tf_labels'])
        lp = m(fc.cuda(), att.cuda(), labels[:, :-1].reshape(fc.shape[0], 2, -1).cuda(), None, mode='forward')
        assert np.abs(lp.cpu().numpy() - g['tf_lp']).max() < LOGP_TOL


def _done(model, B, beam):
    dseq = np.zeros((B, beam, model.seq_length), np.int64)
    dp = np.zeros((B, beam))
    for i in range(B):
        for j, rec in enumerate(model.done_beams[i]):
            L = rec['seq'].shape[0]
            dseq[i, j, :L] = rec['seq'].cpu().numpy()
            dp[i, j] = rec['p']
    return dseq, dp


@pytest.mark.parametrize('mode', PARITY_MODES)
@pytest.mark.parametrize('case', ['beam_wu', 'beam_constraint', 'beam_masked', 'dbs'])
def test_beam_goldens(mode, case):
    g, m, fam, fc, att, masks, T = _small(mode)
    opt = {'beam_size': 4, 'sample_n': 1}
    if case == 'beam_wu':
        opt['length_penalty'] = 'wu_0.5'
    elif case == 'beam_constraint':
        opt['decoding_constraint'] = 1
    elif case == 'dbs':
        opt = {'beam_size': 6, 'group_size': 3, 'diversity_lambda': 0.5, 'sample_n': 1}
    mk = masks.cuda() if case == 'beam_masked' else None
    with torch.no_grad():
        seq, lp = m(fc.cuda(), att.cuda(), mk, opt=opt, mode='sample')
    beam = opt['beam_size']
    assert np.array_equal(seq.cpu().numpy(), g[case + '_seq'])
    dseq, dp = _done(m, fc.shape[0], beam)
    assert np.array_equal(dseq, g[case + '_done_seq'])
    assert np.abs(dp - g[case + '_done_p']).max() < 1e-3
    for j, rec in enumerate(m.done_beams[0]):
        L = rec['logps'].shape[0]
        mine, ref = rec['logps'].cpu().numpy(), g[case + '_logps0'][j, :L]
        assert np.array_equal(np.isneginf(mine), np.isneginf(ref))          # decoding_constraint's -inf entries
        fin = np.isfinite(ref)
        assert np.abs(mine[fin] - ref[fin]).max() < LOGP_TOL


@pytest.mark.parametrize('mode', PARITY_MODES)
def test_sampling_options(mode):
    """top-k, nucleus and block_trigrams sampling: every drawn word is admissible under the oracle's log-probs of the same prefix, and the
    returned rows are those log-probs (block_trigrams rows carry the reference's 2 ln 2 edits, so only their picked entries are compared)."""
    g, m, fam, fc, att, masks, T = _small(mode)
    B = fc.shape[0]
    torch.manual_seed(3)
    with torch.no_grad():
        for method in ('top3', 'top0.8'):
            seq, lp = m(fc.cuda(), att.cuda(), None, opt={'sample_method': method, 'sample_n': 2}, mode='sample')
            seq, lp = seq.cpu(), lp.cpu()
            labels = torch.cat([torch.zeros(2 * B, 1, dtype=torch.long), seq[:, :-1]], 1)
            olp = co.forward_teacher(fam, fc, att, labels.reshape(B, 2, T))
            valid = torch.cat([torch.ones(2 * B, 1, dtype=torch.bool), seq[:, :-1] > 0], 1)
            assert float(((lp - olp).abs().amax(2) * valid).max()) < LOGP_TOL
            rank = (olp > olp.gather(2, seq.unsqueeze(2))).sum(2)
            if method == 'top3':
                assert bool((rank[valid] < 3).all())
            else:
                sp = olp.exp().sort(2, descending=True).values.cumsum(2)
                before = sp.gather(2, (rank - 1).clamp(min=0).unsqueeze(2)).squeeze(2) * (rank > 0)
                assert bool((before[valid] < 0.8 + 1e-4).all())
        seq, lp = m(fc.cuda(), att.cuda(), None, opt={'sample_method': 'sample', 'block_trigrams': 1}, mode='sample')
        assert torch.isfinite(lp.gather(2, seq.unsqueeze(2))).all()


@pytest.mark.parametrize('mode', PARITY_MODES)
def test_recipe_size_beam_golden(mode):
    """a2i2 recipe size (V 9487, E = H = A = 512, T 20), batch 32, beam 5 against the live reference, tie-aware."""
    g = np.load(os.path.join(GOLD, 'att2in2_b32.npz'))
    dims = tuple(int(x) for x in g['cfg'])
    V, E, H, A, F_fc, F_att, T = dims
    B, R, beam, seed = (int(x) for x in g['meta'])
    m = _model(co.make_weights('att2in2', V, E, H, A, F_fc, F_att, seed=seed, logit_scale=12.0), dims, mode)
    fc, att = co.make_inputs(B, R, F_fc, F_att, seed=seed)
    with torch.no_grad():
        seq, lp = m(fc.cuda(), att.cuda(), None, opt={'beam_size': beam, 'sample_n': 1}, mode='sample')
    dseq, dp = _done(m, B, beam)
    decisive = g['image_margin'] > 10 * LOGP_TOL
    same = (dseq == g['done_seq'].astype(np.int64)).all((1, 2))
    assert same[decisive].all(), np.nonzero(decisive & ~same)[0][:8]
    assert same.mean() >= 0.9 and np.abs(dp[same] - g['done_p'][same]).max() < 1e-3


# ---- training steps ------------------------------------------------------------------------------------------------------------------

def _pair(mode, seed=31):
    W = co.make_weights('att2in2', CFG['V'], CFG['E'], CFG['H'], CFG['A'], CFG['F_fc'], CFG['F_att'], seed=seed, logit_scale=5.0)
    m = _model(W, tuple(CFG[k] for k in ('V', 'E', 'H', 'A', 'F_fc', 'F_att', 'T')), mode)
    return m, W


def _check_grads(model, grads, ograds, rel=5e-4):
    name_of = {id(p): k for k, p in model.state_dict(keep_vars=True).items()}
    assert len(grads) == 17
    for p, g in grads.items():
        key = name_of[id(p)]
        ref = ograds[key]
        scale = float(ref.abs().max())
        err = float((g.cpu() - ref).abs().max())
        assert err <= rel * scale + 2e-9, (key, err, scale)
    assert sum(float(v.abs().max()) > 1e-6 for v in ograds.values()) >= 15


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
@pytest.mark.parametrize('kind', ['greedy', 'leave_one_out', 'keep_rows'])
def test_scst_step(mode, kind):
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    model, W = _pair(mode)
    B, R, n, T, p, seed = 5, 11, 4, CFG['T'], 0.5, 1234
    fc, att = co.make_inputs(B, R, CFG['F_fc'], CFG['F_att'], seed=4)
    regions = torch.ones(B, R)
    regions[2, 6:] = 0
    gts = cdo.make_refs(B, CFG['V'], seed=2)
    df, ref_len = cdo.build_document_frequency(cdo.make_refs(200, CFG['V'], seed=4))
    table = b200.rewards.CiderDTable(df, ref_len)
    model.train()
    keep = 13 if kind == 'keep_rows' else 0
    res = model.scst_step(fc.cuda(), att.cuda(), gts, table, n, drop_prob=p, seed=seed, att_masks=regions.cuda(),
                          baseline='leave_one_out' if kind == 'leave_one_out' else 'greedy', keep_rows=keep)
    torch.cuda.synchronize()
    sseq = res['sample_seq'].cpu()
    Wg = {k: v.clone().requires_grad_(True) for k, v in W.items()}
    fam = ao.Att2in2Family(Wg, T)
    if kind == 'leave_one_out':
        sc = cdo.get_scores(gts, sseq.numpy(), df, ref_len).reshape(B, n)
        reward = torch.from_numpy(np.repeat((sc - (sc.sum(1, keepdims=True) - sc) / (n - 1)).reshape(-1, 1), T, 1)).float()
    else:
        og, _ = co.sample(ao.Att2in2Family(W, T), fc, att, regions)
        assert torch.equal(res['greedy_seq'].cpu(), og)
        reward, _ = cdo.self_critical_reward(og.numpy(), gts, sseq.numpy(), df, ref_len)
        reward = torch.from_numpy(reward).float()
    fam.drop = att2in2_masks(b200, seed, p, B, R, B * n, T, CFG['E'], CFG['H'])
    _, lp = co.sample(fam, fc, att, regions, sample_method='sample', sample_n=n, forced_tokens=sseq)
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


@pytest.mark.parametrize('mode', PARITY_MODES)
@pytest.mark.parametrize('ss_prob', [0.0, 0.4])
def test_xe_step(mode, ss_prob):
    """XE with dropout and region masks; with ss_prob > 0 the oracle is fed the words the engine actually used."""
    import imagecaptioning.pytorch_b200 as b200
    model, W = _pair(mode, seed=21)
    B, R, spi, T, p, seed = 6, 9, 5, CFG['T'], 0.0 if ss_prob else 0.5, 991
    fc, att = co.make_inputs(B, R, CFG['F_fc'], CFG['F_att'], seed=4)
    regions = torch.ones(B, R)
    regions[0, 4:] = 0
    labels, masks = _labels(B, spi, CFG['V'], T + 2, seed=12)
    model.train()
    model.ss_prob = ss_prob
    res = model.xe_step(fc.cuda(), att.cuda(), labels.cuda(), masks.cuda(), label_smoothing=0.1, drop_prob=p, seed=seed, att_masks=regions.cuda())
    model.ss_prob = 0.0
    torch.cuda.synchronize()
    used = res['tokens_used'].cpu().reshape(B, spi, -1) if ss_prob else labels[..., :-1]
    if ss_prob:
        assert bool((used != labels[..., :-1]).any())
    Wg = {k: v.clone().requires_grad_(True) for k, v in W.items()}
    fam = ao.Att2in2Family(Wg, T)
    if p:
        fam.drop = att2in2_masks(b200, seed, p, B, R, B * spi, T + 1, CFG['E'], CFG['H'])
    lp = co.forward_teacher(fam, fc, att, used, regions)
    loss = co.label_smoothing_loss(lp, labels[..., 1:], masks[..., 1:], 0.1)
    loss.backward()
    steps = lp.shape[1]
    assert float((res['logprobs'].cpu() - lp.detach())[:, :steps].abs().max()) < LOGP_TOL
    assert abs(float(res['loss']) - float(loss)) < LOGP_TOL
    _check_grads(model, res['grads'], {k: v.grad for k, v in Wg.items()})


def test_step_graph_replay_identical():
    """Eager (first call), captured (second) and replayed (third) SCST steps with the same seed draw the same samples and loss."""
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    model, _ = _pair('tc_f16x3')
    B, R, n = 4, 7, 3
    fc, att = co.make_inputs(B, R, CFG['F_fc'], CFG['F_att'], seed=5)
    gts = cdo.make_refs(B, CFG['V'], seed=3)
    table = b200.rewards.CiderDTable(*cdo.build_document_frequency(cdo.make_refs(100, CFG['V'], seed=4)))
    model.train()
    outs = []
    for _ in range(3):
        res = model.scst_step(fc.cuda(), att.cuda(), gts, table, n, drop_prob=0.5, seed=77)
        outs.append({'loss': res['loss'].clone(), 'seq': res['sample_seq'].clone(), 'g': [g.clone() for g in res['grads'].values()]})
    for o in outs[1:]:
        assert torch.equal(o['loss'], outs[0]['loss']) and torch.equal(o['seq'], outs[0]['seq'])
        for a, b in zip(o['g'], outs[0]['g']):          # the embedding and alpha_net gradients accumulate with atomics: not bit-reproducible
            assert float((a - b).abs().max()) <= 1e-5 * float(b.abs().max()) + 1e-9
    res = model.scst_step(fc.cuda(), att.cuda(), gts, table, n, drop_prob=0.5, seed=78)      # a new seed replays with new draws
    assert not torch.equal(res['sample_seq'], outs[0]['seq'])


@pytest.mark.parametrize('branch', ['sc', 'struc'])
def test_loss_wrapper_backward_and_adam(branch):
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    model, _ = _pair('tc_f16x3')
    B, R, n = 4, 7, 3
    fc, att = co.make_inputs(B, R, CFG['F_fc'], CFG['F_att'], seed=5)
    gts = cdo.make_refs(B, CFG['V'], seed=3)
    b200.rewards.reset_scorer()
    b200.rewards.init_scorer(b200.rewards.CiderDTable(*cdo.build_document_frequency(cdo.make_refs(100, CFG['V'], seed=4))))
    opt = argparse.Namespace(sc_sample_method='greedy', sc_beam_size=1, train_sample_method='sample', train_beam_size=1, train_sample_n=n,
                             cider_reward_weight=1, bleu_reward_weight=0, structure_loss_type='new_self_critical', structure_loss_weight=1.0,
                             label_smoothing=0.0)
    lw = b200.B200LossWrapper(model, opt)
    labels, masks = _labels(B, n, CFG['V'], CFG['T'] + 2, seed=2)
    optim = b200.optim.FusedAdam(model.parameters(), lr=1e-3)
    before = {k: v.detach().clone() for k, v in model.state_dict().items()}
    for _ in range(2):
        optim.zero_grad()
        out = lw(fc.cuda(), att.cuda(), labels.cuda(), masks.cuda(), None, gts, torch.arange(B), branch == 'sc', branch == 'struc', False)
        assert out['loss'].requires_grad and torch.isfinite(out['loss'])
        out['loss'].backward()
        assert all(p.grad is not None for p in model.parameters())
        optim.step()                      # changes the weights: the next call re-binds them
    assert any(not torch.equal(before[k], v) for k, v in model.state_dict().items())
    b200.rewards.reset_scorer()


@pytest.mark.parametrize('method', ['bs', 'dbs'])
def test_eval_split_n(method):
    from imagecaptioning.pytorch_b200 import eval_utils
    from imagecaptioning.pytorch_b200.utils import decode_sequence
    g, m, fam, fc, att, masks, T = _small('simt_fp32')
    B = fc.shape[0]
    preds = []
    data = {'infos': [{'id': 100 + i} for i in range(B)]}
    eval_utils.eval_split_n(m, preds, (fc.cuda(), att.cuda(), None, data), {'sample_n_method': method, 'sample_n': 3, 'beam_size': 3, 'verbose': False})
    assert len(preds) == 3 * B
    if method == 'dbs':
        _, _, done = dbs_oracle.diverse_sample_beam(fam, fc, att, beam_size=9, group_size=3, diversity_lambda=0.5)
        picks = (0, 3, 6)
    else:
        _, _, done = co.sample_beam(fam, fc, att, beam_size=3, sample_n=3)
        picks = (0, 1, 2)
    want = []
    for k in range(B):
        for sent in decode_sequence(m.vocab, torch.stack([done[k][j]['seq'] for j in picks])):
            want.append({'image_id': 100 + k, 'caption': sent})
    assert preds == want
