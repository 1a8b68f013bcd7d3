"""Diverse beam search (group_size > 1) on the engine, UpDown and AoANet: the reference goldens (tests/make_dbs_golden.py), the restatement in
dbs_oracle, and the invariants that tie it to the plain beam search."""
import json
import os

import numpy as np
import pytest
import torch

from helpers import LOGP_TOL, build_pair, co
import dbs_oracle

pytestmark = pytest.mark.gpu

CONFIGS = [('updown', 'simt_fp32'), ('updown', 'tc_f16x3'), ('aoa', 'tc_f16x3')]
P_TOL = 1e-4
DECISIVE = 5 * LOGP_TOL       # an image's decisions count as ties below this candidate gap (log-prob units)


def _small(golden_dir):
    g = np.load(os.path.join(golden_dir, 'dbs_small.npz'))
    cfg = dict(zip(('V', 'E', 'H', 'A', 'F_fc', 'F_att', 'T'), (int(x) for x in g['cfg'])))
    return g, cfg, json.loads(str(g['cases'])), json.loads(str(g['meta']))


def _pair(family, mode, cfg, meta):
    m = meta[family]
    model, fam = build_pair(family, seed=m['seed'], logit_scale=m['logit_scale'], mode=mode, heads=4, **cfg)
    fc, att = co.make_inputs(m['B'], m['R'], cfg['F_fc'], cfg['F_att'], seed=m['seed'])
    masks = torch.ones(m['B'], m['R'])
    masks[1, 5:] = 0
    masks[3, 3:] = 0
    return model, fam, fc, att, masks


def _opt(case):
    return dict({'beam_size': case['beam_size'], 'group_size': case['group_size'], 'diversity_lambda': case['diversity_lambda'], 'sample_n': 1},
                **case['opts'])


def _done(model, B, n):
    seqs = np.zeros((B, n, model.seq_length), np.int64)
    ps = np.zeros((B, n))
    for i in range(B):
        for j in range(n):
            rec = model.done_beams[i][j]
            seqs[i, j, :len(rec['seq'])] = rec['seq'].cpu().numpy()
            ps[i, j] = rec['p']
    return seqs, ps


@pytest.mark.parametrize('family,mode', CONFIGS)
def test_dbs_small_goldens(golden_dir, family, mode):
    """Every golden case: ids bit-exact where the decision is not a numerical tie, picked log-probs and record scores within 1e-4, done_beams
    in group order, and the full log-prob rows of materialised records within 1e-4."""
    g, cfg, cases, meta = _small(golden_dir)
    model, fam, fc, att, masks = _pair(family, mode, cfg, meta)
    B = fc.shape[0]
    n_images, n_decisive = 0, 0
    for case in cases:
        key = '%s_%s_' % (family, case['name'])
        margins = []
        oo = case['opts']
        dbs_oracle.diverse_sample_beam(fam, fc, att, masks if case['masked'] else None, beam_size=case['beam_size'], group_size=case['group_size'],
                                       diversity_lambda=case['diversity_lambda'], length_penalty=oo.get('length_penalty', ''),
                                       temperature=oo.get('temperature', 1.0), decoding_constraint=bool(oo.get('decoding_constraint', 0)),
                                       margin_rows=margins)
        decisive = (torch.stack(margins, 1).min(1).values > DECISIVE).numpy()     # per image: every group step clear of a tie
        with torch.no_grad():
            seq, lp = model(fc.cuda(), att.cuda(), masks.cuda() if case['masked'] else None, opt=_opt(case), mode='sample')
        n = case['beam_size']
        dseq, dp = _done(model, B, n)
        assert np.abs(dp - g[key + 'done_p']).max() < P_TOL, (case['name'], np.abs(dp - g[key + 'done_p']).max())
        n_images += B
        n_decisive += int(decisive.sum())
        seq_c = seq.cpu().numpy()
        assert np.array_equal(seq_c[:B][decisive], g[key + 'seq'][:B][decisive]), case['name']
        assert np.array_equal(dseq[decisive], g[key + 'done_seq'][decisive]), case['name']
        picked = lp.gather(2, seq.unsqueeze(2)).squeeze(2).cpu().numpy()
        assert np.abs(picked[:B][decisive] - g[key + 'picked'][:B][decisive]).max(initial=0.0) < LOGP_TOL, case['name']
        if decisive[0]:
            for j in range(n):
                rec = model.done_beams[0][j]
                L = len(rec['seq'])
                np.testing.assert_allclose(rec['logps'].cpu().numpy(), g[key + 'logps0'][j, :L], rtol=0, atol=LOGP_TOL,
                                           err_msg='%s %d' % (case['name'], j))
        if case['opts'].get('sample_n', 1) > 1:
            assert seq.shape[0] == B * case['opts']['sample_n'] and not seq[B:].any() and not lp[B:].any()
    assert n_decisive >= 0.75 * n_images, (n_decisive, n_images)
    print('%s [%s]: %d / %d (case, image) pairs decisive and bit-exact' % (family, mode, n_decisive, n_images))


@pytest.mark.parametrize('family,mode', CONFIGS)
def test_dbs_lambda_zero_is_plain_beam_per_group(golden_dir, family, mode):
    """With diversity_lambda = 0 the groups do not interact: every group's done_beams equal a plain beam search of width bdash."""
    g, cfg, _, meta = _small(golden_dir)
    model, _, fc, att, _ = _pair(family, mode, cfg, meta)
    B = fc.shape[0]
    fcd, attd = fc.cuda(), att.cuda()
    with torch.no_grad():
        model(fcd, attd, None, opt={'beam_size': 2, 'sample_n': 1}, mode='sample')
        pseq, pp = _done(model, B, 2)
        model(fcd, attd, None, opt={'beam_size': 6, 'group_size': 3, 'diversity_lambda': 0.0, 'sample_n': 1}, mode='sample')
        dseq, dp = _done(model, B, 6)
    for grp in range(3):
        assert np.array_equal(dseq[:, 2 * grp:2 * grp + 2], pseq), grp
        assert np.abs(dp[:, 2 * grp:2 * grp + 2] - pp).max() < 1e-5, grp


def _raw_call(model, fc, att, masks, beam, group_size, lam, fn):
    """Calls a beam entry point through the C ABI directly (group_size 1 never reaches capb200_*_diverse from Python)."""
    from imagecaptioning.pytorch_b200 import _lib
    lib = model._ensure_engine(fc.device)
    B, T = fc.shape[0], model.seq_length
    V1 = model.vocab_size + 1
    seq = torch.empty(B, T, dtype=torch.long, device=fc.device)
    lp = torch.empty(B, T, V1, device=fc.device)
    d_seq = torch.empty(B, beam, T, dtype=torch.long, device=fc.device)
    d_len = torch.empty(B, beam, dtype=torch.int32, device=fc.device)
    d_p = torch.empty(B, beam, device=fc.device)
    d_raw = torch.empty(B, beam, device=fc.device)
    bo = _lib.BeamOpts(beam, 1, 0, 0.0, 1.0, _lib.DecodeEdits.none())
    R = att.shape[1]
    if fn == 'plain':
        rc = model._call_beam(lib, fc, att, masks, B, R, bo, seq, lp, d_seq, d_len, d_p, d_raw)
    else:
        rc = model._call_beam_diverse(lib, fc, att, masks, B, R, _lib.DiverseOpts(bo, group_size, lam), seq, lp, d_seq, d_len, d_p, d_raw)
    _lib.check(rc, fn)
    return seq, lp, d_seq, d_p


@pytest.mark.parametrize('family,mode', CONFIGS)
def test_dbs_group_size_one_is_plain_beam(golden_dir, family, mode):
    g, cfg, _, meta = _small(golden_dir)
    model, _, fc, att, _ = _pair(family, mode, cfg, meta)
    fcd, attd = fc.cuda(), att.cuda()
    with torch.no_grad():
        a = _raw_call(model, fcd, attd, None, 4, 1, 0.5, 'plain')
        b = _raw_call(model, fcd, attd, None, 4, 1, 0.5, 'diverse')
    for x, y in zip(a, b):
        assert torch.equal(x, y)


@pytest.mark.parametrize('family,mode', CONFIGS)
def test_dbs_replay_and_alternation(golden_dir, family, mode, monkeypatch, capfd):
    """The beam loop is run eagerly the first time a configuration is seen, captured into a CUDA graph the second time in a row and replayed
    from then on; the engine keeps one captured loop.  Three identical diverse calls (eager, capture, replay) agree bit for bit, and so do
    the captures and replays of the next configurations: a lambda change, a plain beam search of the same batch and width, and the first
    configuration again.  The first call after each switch must not replay the previous configuration's graph, which the graph debug
    messages confirm together with the results.  The calls run on a side stream: torch's legacy default stream cannot be captured, and
    on it the engine runs every beam loop eagerly."""
    g, cfg, _, meta = _small(golden_dir)
    model, _, fc, att, _ = _pair(family, mode, cfg, meta)
    fcd, attd = fc.cuda(), att.cuda()
    B = fc.shape[0]
    opts = {'dbs': {'beam_size': 6, 'group_size': 3, 'diversity_lambda': 2.0, 'sample_n': 1},
            'dbs2': {'beam_size': 6, 'group_size': 3, 'diversity_lambda': 0.5, 'sample_n': 1},
            'plain': {'beam_size': 6, 'sample_n': 1}}
    # (configuration, what the loop does on this call)
    calls = [('dbs', 'eager'), ('dbs', 'captured'), ('dbs', 'replayed'),
             ('dbs2', 'eager'), ('dbs2', 'captured'), ('dbs2', 'replayed'),
             ('plain', 'eager'), ('plain', 'captured'), ('plain', 'replayed'),
             ('dbs', 'eager'), ('dbs', 'captured'), ('dbs', 'replayed')]
    monkeypatch.setenv('CAPB200_GRAPH_DEBUG', '1')
    first = {}
    capfd.readouterr()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.no_grad(), torch.cuda.stream(side):
        for i, (name, how) in enumerate(calls):
            seq, lp = model(fcd, attd, None, opt=opts[name], mode='sample')
            dseq, dp = _done(model, B, 6)
            out = (seq.cpu().clone(), lp.gather(2, seq.unsqueeze(2)).squeeze(2).cpu().clone(), dseq, dp)
            err = capfd.readouterr().err
            seen = 'replayed' if 'beam loop replayed' in err else ('captured' if 'beam loop captured' in err else 'eager')
            assert seen == how, (i, name, how, err)
            if name not in first:
                first[name] = out
                continue
            ref = first[name]
            assert torch.equal(ref[0], out[0]) and torch.equal(ref[1], out[1]), (i, name, how)
            assert np.array_equal(ref[2], out[2]) and np.array_equal(ref[3], out[3]), (i, name, how)
    assert not np.array_equal(first['dbs'][2], first['plain'][2])
    assert not np.array_equal(first['dbs'][3], first['dbs2'][3])


def test_eval_split_n_dbs_matches_restatement(golden_dir):
    """eval_split_n(sample_n_method='dbs', sample_n=3, beam_size=3): three captions per image, each group's best, as the restatement gives."""
    from imagecaptioning.pytorch_b200 import eval_utils
    from imagecaptioning.pytorch_b200.utils import decode_sequence
    g, cfg, _, meta = _small(golden_dir)
    model, fam, fc, att, _ = _pair('updown', 'simt_fp32', cfg, meta)
    B = fc.shape[0]
    preds = []
    data = {'infos': [{'id': 100 + i} for i in range(B)]}
    eval_utils.eval_split_n(model, preds, (fc.cuda(), att.cuda(), None, data), {'sample_n_method': 'dbs', 'sample_n': 3, 'beam_size': 3, 'verbose': False})
    assert len(preds) == 3 * B
    _, _, done = dbs_oracle.diverse_sample_beam(fam, fc, att, beam_size=9, group_size=3, diversity_lambda=0.5)
    want = []
    for k in range(B):
        for sent in decode_sequence(model.vocab, torch.stack([done[k][j]['seq'] for j in (0, 3, 6)])):
            want.append({'image_id': 100 + k, 'caption': sent})
    assert preds == want


def test_updown_dbs_config_dims_golden(golden_dir):
    """BASELINE configs[1] dimensions, batch 32, beam 9 in 3 groups, against the live reference: record scores everywhere, bit-exact ids on
    every image whose decisions are not numerical ties."""
    path = os.path.join(golden_dir, 'updown_dbs_b32.npz')
    g = np.load(path)
    cfg = dict(zip(('V', 'E', 'H', 'A', 'F_fc', 'F_att', 'T'), (int(x) for x in g['cfg'])))
    B, R, beam, G, seed = (int(x) for x in g['meta'])
    model, _ = build_pair('updown', seed=seed, logit_scale=12.0, mode='tc_f16x3', **cfg)
    fc, att = co.make_inputs(B, R, cfg['F_fc'], cfg['F_att'], seed=seed)
    with torch.no_grad():
        seq, lp = model(fc.cuda(), att.cuda(), None, opt={'beam_size': beam, 'group_size': G, 'diversity_lambda': float(g['diversity_lambda']),
                                                          'sample_n': 1}, mode='sample')
    dseq, dp = _done(model, B, beam)
    decisive = g['image_margin'] > 10 * LOGP_TOL
    same = (dseq == g['done_seq'].astype(np.int64)).all((1, 2))
    assert same[decisive].all(), np.nonzero(decisive & ~same)[0][:8]
    assert same.mean() >= 0.9, same.mean()
    assert np.abs(dp[same] - g['done_p'][same]).max() < 1e-3
    picked = lp.gather(2, seq.unsqueeze(2)).squeeze(2).cpu().numpy()
    s0 = (seq.cpu().numpy() == g['seq'].astype(np.int64)).all(1)
    assert np.abs(picked[s0] - g['picked'][s0]).max() < LOGP_TOL
    print('updown DBS B=32 beam 9 G=3: %.1f %% of the images bit-exact (%d decisive)' % (100 * same.mean(), int(decisive.sum())))
