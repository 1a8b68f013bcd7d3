"""Test-time ensembles on the GPU: every mix x weight set x case of the reference's AttEnsemble goldens, sampling invariants, the one-member
identity, the beam loop's CUDA graph, and one UpDown pair at BASELINE.json configs[1] dimensions."""
import json
import os

import numpy as np
import pytest
import torch

from helpers import LOGP_TOL, co, family_opt
import dbs_oracle
import ensemble_oracle as eo

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ensemble_small.npz')
GAP = 1e-2           # token ids must be bit-exact wherever the winner / runner-up gap exceeds this
MODES = ['tc_f16x3', 'simt_fp32']


def _golden():
    g = np.load(GOLD)
    return g, json.loads(str(g['meta']))


G, META = _golden()
CASES = {name: (opts, masked) for name, opts, masked in META['cases']}


def engine_members(meta, mix, mode):
    import imagecaptioning.pytorch_b200 as b200
    c = meta['cfg']
    out = []
    for f, W in eo.member_weight_dicts(meta, mix):
        m = b200.setup(family_opt(f, c['V'], c['E'], c['H'], c['A'], c['F_fc'], c['F_att'], c['T'], heads=meta['aoa_heads']), numeric_mode=mode)
        m.load_state_dict(W, strict=True)
        out.append(m.cuda().eval())
    return out


def ensemble(meta, mix, wname, mode):
    import imagecaptioning.pytorch_b200 as b200
    return b200.B200AttEnsemble(engine_members(meta, mix, mode), weights=eo.mix_weights(meta, mix, wname))


def inputs(meta):
    c = meta['cfg']
    return co.make_inputs(meta['B'], meta['R'], c['F_fc'], c['F_att'], seed=meta['input_seed'])


def close_rows(mine, ref, atol):
    """|mine - ref| per row (max over the trailing axes), with equal -inf patterns required (decode edits)."""
    mine, ref = np.asarray(mine), np.asarray(ref)
    assert np.array_equal(np.isneginf(mine), np.isneginf(ref))
    d = np.where(np.isfinite(ref), np.abs(np.where(np.isfinite(mine), mine, 0) - np.where(np.isfinite(ref), ref, 0)), 0)
    return d.reshape(d.shape[0], int(np.prod(d.shape[1:]))).max(1, initial=0.0) < atol


def greedy_gaps(seq, lp):
    """Per row: the smallest top-1 / top-2 gap of the reference's log-prob rows over the steps that chose a word."""
    alive = torch.cat([torch.ones(seq.shape[0], 1, dtype=torch.bool), (seq[:, :-1] > 0).cumprod(1).bool()], 1)
    top2 = lp.topk(2, dim=2).values
    return (top2[..., 0] - top2[..., 1]).masked_fill(~alive, float('inf')).min(1).values.numpy()


def check_decode(fam, fc, att, masks, seq, lp, strict, ref_seq, ref_lp):
    """The suite's bar: rows decided by more than GAP everywhere must equal the reference's ids and log-prob rows (within 1e-4); every returned
    caption, re-scored by teacher forcing on the restatement, carries the log-probs the engine reported."""
    assert np.array_equal(seq.numpy()[strict], ref_seq[strict])
    assert close_rows(lp.numpy()[strict], ref_lp[strict], LOGP_TOL).all()
    N, T = seq.shape
    B = fc.shape[0]
    labels = torch.cat([torch.zeros(N, 1, dtype=torch.long), seq[:, :-1]], 1).reshape(B, N // B, T)
    tf = co.forward_teacher(fam, fc, att, labels, None if masks is None else masks.cpu())
    valid = torch.cat([torch.ones(N, 1, dtype=torch.bool), (seq[:, :-1] > 0).cumprod(1).bool()], 1)
    mine, theirs = lp.gather(2, seq.unsqueeze(2)).squeeze(2), tf.gather(2, seq.unsqueeze(2)).squeeze(2)
    assert float(((mine - theirs).abs() * valid).max()) < 2 * LOGP_TOL


@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('case', list(CASES))
@pytest.mark.parametrize('wname', list(META['weights']))
@pytest.mark.parametrize('mix', list(META['mixes']))
def test_ensemble_matches_reference(mix, wname, case, mode):
    meta, c = META, META['cfg']
    opts, masked = CASES[case]
    key = '%s_%s_%s_' % (mix, wname, case)
    fc, att = inputs(meta)
    masks = eo.case_masks(meta['B'], meta['R']).cuda() if masked else None
    ens = ensemble(meta, mix, wname, mode)
    with torch.no_grad():
        if opts == 'teacher':
            lab = eo.labels(meta['B'], c['T'], c['V'], meta['label_seed']).cuda()
            out = ens(fc.cuda(), att.cuda(), lab, masks).cpu().numpy()
            assert close_rows(out, G[key + 'out'], LOGP_TOL).all()
            return
        seq, lp = ens(fc.cuda(), att.cuda(), masks, opt=dict(opts), mode='sample')
    fam = eo.oracle_for(meta, mix, wname)
    seq, lp = seq.cpu(), lp.cpu()
    if opts.get('beam_size', 1) > 1:
        margins = []
        eo.run_oracle(fam, fc, att, meta, opts, masked, margins=margins)
        gap = torch.stack(margins, 1).min(1).values.numpy()
    else:
        gap = greedy_gaps(torch.from_numpy(G[key + 'seq']), torch.from_numpy(G[key + 'logprobs']))
    strict = gap > GAP
    check_decode(fam, fc, att, masks, seq, lp, strict, G[key + 'seq'], G[key + 'logprobs'])
    if opts.get('beam_size', 1) > 1:
        b = opts['beam_size']
        done = ens.done_beams
        dseq, dlen, dp = dbs_oracle.beams_to_arrays([[{'seq': r['seq'].cpu(), 'p': r['p']} for r in img] for img in done], b, c['T'])
        assert np.array_equal(dseq[strict], G[key + 'done_seq'][strict]) and np.array_equal(dlen[strict], G[key + 'done_len'][strict])
        assert np.abs(dp[strict] - G[key + 'done_p'][strict]).max(initial=0.0) < LOGP_TOL
        assert np.abs(dp[:, 0] - G[key + 'done_p'][:, 0]).max() < 1e-3          # a near-tie may swap the winner, never worsen it
        for i in range(meta['B']):           # done_beams[i][0]['logps'] are the rows of seq[i]
            L = int(dlen[i, 0])
            assert close_rows(done[i][0]['logps'].cpu().numpy()[None], lp.numpy()[i:i + 1, :L], 1e-6).all()


@pytest.mark.parametrize('method', ['sample', 'top3', 'top0.8'])
@pytest.mark.parametrize('mix', ['mixed3', 'newfc_updown'])
def test_sampling_invariants_and_teacher_forcing(mix, method):
    """Draws cannot be compared with the reference's random stream: check what holds for every draw, then re-score the drawn captions by
    teacher forcing on the restatement."""
    meta, c = META, META['cfg']
    fc, att = inputs(meta)
    ens = ensemble(meta, mix, 'uneq', 'tc_f16x3')
    torch.manual_seed(5)
    with torch.no_grad():
        seq, lp = ens(fc.cuda(), att.cuda(), None, opt={'sample_method': method, 'beam_size': 1, 'sample_n': 2, 'temperature': 0.9}, mode='sample')
    seq, lp = seq.cpu(), lp.cpu()
    N, T = seq.shape
    assert N == 2 * meta['B'] and lp.shape == (N, T, c['V'] + 1)
    assert int(seq.min()) >= 0 and int(seq.max()) <= c['V']
    alive = torch.cat([torch.ones(N, 1, dtype=torch.bool), (seq[:, :-1] > 0).cumprod(1).bool()], 1)
    assert not bool(seq[~alive].any()), 'a token after the end of a caption'
    assert bool((lp[~alive] == 0).all()), 'finished rows carry zero log-prob rows'
    lse = torch.logsumexp(lp, 2)
    assert float(lse[alive].abs().max()) < 1e-4, 'every live row is a normalised log-distribution'
    labels = torch.cat([torch.zeros(N, 1, dtype=torch.long), seq[:, :-1]], 1).reshape(meta['B'], 2, T)
    tf = co.forward_teacher(eo.oracle_for(meta, mix, 'uneq'), fc, att, labels)
    picked, theirs = lp.gather(2, seq.unsqueeze(2)).squeeze(2), tf.gather(2, seq.unsqueeze(2)).squeeze(2)
    assert float(((picked - theirs).abs() * alive).max()) < 2 * LOGP_TOL


@pytest.mark.parametrize('family', ['updown', 'att2in2', 'newfc', 'aoa'])
def test_one_member_ensemble_is_the_single_model(family):
    import imagecaptioning.pytorch_b200 as b200
    c = META['cfg']
    W = co.make_weights(family, c['V'], c['E'], c['H'], c['A'], c['F_fc'], c['F_att'], seed=31, logit_scale=META['logit_scale'])
    m = b200.setup(family_opt(family, c['V'], c['E'], c['H'], c['A'], c['F_fc'], c['F_att'], c['T'], heads=META['aoa_heads']))
    m.load_state_dict(W, strict=True)
    m = m.cuda().eval()
    ens = b200.B200AttEnsemble([m], weights=[2.0])
    fc, att = (x.cuda() for x in inputs(META))
    with torch.no_grad():
        for opt in ({'sample_method': 'greedy', 'beam_size': 1}, {'beam_size': 3, 'sample_n': 3}):
            s1, l1 = m(fc, att, None, opt=opt, mode='sample')
            s2, l2 = ens(fc, att, None, opt=opt, mode='sample')
            assert torch.equal(s1, s2), (opt, s1, s2)
            fin = torch.isfinite(l1)
            assert torch.equal(fin, torch.isfinite(l2)) and float((l1[fin] - l2[fin]).abs().max()) < 1e-5, opt


def test_beam_loop_graph_eager_captured_replayed():
    """First call eager, second captured into a CUDA graph, third replayed: identical outputs and launch counts.  A changed weight value is
    a different configuration (the weights are arguments of the captured mixing launches) and is never replayed from the old graph."""
    fc, att = (x.cuda() for x in inputs(META))
    ens = ensemble(META, 'mixed3', 'uneq', 'tc_f16x3')
    opt = {'beam_size': 5, 'sample_n': 1, 'length_penalty': 'wu_0.5', 'decoding_constraint': 1}
    outs, counts = [], []
    with torch.no_grad():
        for _ in range(3):
            before = ens.launch_count
            seq, lp = ens(fc, att, None, opt=opt, mode='sample')
            torch.cuda.synchronize()
            counts.append(ens.launch_count - before)
            outs.append((seq.clone(), lp.clone(), ens.done_beams[1][2]['p']))
        assert counts[0] == counts[1] == counts[2] > 0, counts
        for seq, lp, p in outs[1:]:
            assert torch.equal(seq, outs[0][0]) and torch.equal(lp, outs[0][1]) and p == outs[0][2]
        ens.weights.copy_(torch.tensor([1.0, 1.0, 1.0]))
        seq, lp = ens(fc, att, None, opt=opt, mode='sample')
        ref = ensemble(META, 'mixed3', 'eq', 'tc_f16x3')
        rseq, rlp = ref(fc, att, None, opt=opt, mode='sample')
        assert torch.equal(seq, rseq) and torch.equal(lp, rlp)


def test_cabi_refuses_mismatched_members():
    """Members with another vocab_size or seq_length than the first are refused before any device work of the call."""
    import ctypes
    import imagecaptioning.pytorch_b200 as b200
    from imagecaptioning.pytorch_b200 import _lib
    c = META['cfg']
    fc, att = (x.cuda() for x in inputs(META))
    models = []
    for V, T in ((c['V'], c['T']), (c['V'] + 1, c['T']), (c['V'], c['T'] + 1)):
        m = b200.setup(family_opt('updown', V, c['E'], c['H'], c['A'], c['F_fc'], c['F_att'], T)).cuda().eval()
        m._ensure_engine(fc.device)
        models.append(m)
    lib = _lib.load()
    s = lib.capb200_ensemble_create()
    seq = torch.empty(META['B'], c['T'], dtype=torch.long, device='cuda')
    for other in models[1:]:
        arr = (_lib.EnsembleMember * 2)()
        for k, m in enumerate((models[0], other)):
            arr[k].family, arr[k].engine, arr[k].weight = _lib.FAMILY_UPDOWN, m._engine, 1.0
        bo = _lib.BeamOpts(3, 1)
        rc = lib.capb200_ensemble_decode_beam(s, arr, 2, _lib.ptr(fc), _lib.ptr(att), None, META['B'], META['R'], ctypes.byref(bo), _lib.ptr(seq),
                                              None, None, None, None, None, _lib.current_stream())
        assert rc == 1 and b'vocab_size and seq_length' in lib.capb200_last_error()
    assert lib.capb200_ensemble_launch_count(s) == 0
    lib.capb200_ensemble_destroy(s)


def test_updown_pair_configs1_batch32():
    """Two UpDown members at BASELINE.json configs[1] dimensions (V 9487, H 1000, 36 x 2048 regions, T 20), batch 32, beam 5."""
    import imagecaptioning.pytorch_b200 as b200
    cfg = dict(V=9487, E=1000, H=1000, A=512, F_fc=2048, F_att=2048, T=20)
    B, R, beam = 32, 36, 5
    Ws = [co.make_weights('updown', cfg['V'], cfg['E'], cfg['H'], cfg['A'], cfg['F_fc'], cfg['F_att'], seed=s, logit_scale=12.0) for s in (1234, 1235)]
    members = []
    for W in Ws:
        m = b200.setup(family_opt('updown', *cfg.values()))
        m.load_state_dict(W, strict=True)
        members.append(m.cuda().eval())
    ens = b200.B200AttEnsemble(members, weights=[1.0, 2.0])
    fc, att = co.make_inputs(B, R, cfg['F_fc'], cfg['F_att'], seed=77)
    with torch.no_grad():
        seq, lp = ens(fc.cuda(), att.cuda(), None, opt={'beam_size': beam, 'sample_n': 1}, mode='sample')
        p = np.array([d[0]['p'] for d in ens.done_beams])
        fam = eo.EnsembleFamily([co.Family('updown', W, cfg['T']) for W in Ws], [1.0, 2.0])
        margins = []
        oseq, olp, odone = dbs_oracle.diverse_sample_beam(fam, fc, att, beam_size=beam, group_size=1, margin_rows=margins)
    strict = torch.stack(margins, 1).min(1).values.numpy() > GAP
    check_decode(fam, fc, att, None, seq.cpu(), lp.cpu(), strict, oseq.numpy(), olp.numpy())
    op = np.array([d[0]['p'] for d in odone])
    assert np.abs(p[strict] - op[strict]).max(initial=0.0) < LOGP_TOL and np.abs(p - op).max() < 1e-3
