"""Diverse beam search without a GPU: the restatement in dbs_oracle against the reference goldens, and the option guards."""
import json
import os

import numpy as np
import pytest
import torch

from helpers import co, family_opt, make_opt
import dbs_oracle

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
AOA_HEADS = 4


def _small():
    g = np.load(os.path.join(GOLD, 'dbs_small.npz'))
    return g, json.loads(str(g['cases'])), json.loads(str(g['meta']))


def small_setup(family, g, meta):
    V, E, H, A, F_fc, F_att, T = (int(x) for x in g['cfg'])
    m = meta[family]
    W = co.make_weights(family, V, E, H, A, F_fc, F_att, seed=m['seed'], logit_scale=m['logit_scale'])
    fc, att = co.make_inputs(m['B'], m['R'], F_fc, F_att, seed=m['seed'])
    masks = torch.ones(m['B'], m['R'])
    masks[1, 5:] = 0
    masks[3, 3:] = 0
    return W, fc, att, masks, (V, E, H, A, F_fc, F_att, T)


def oracle_case(fam, fc, att, masks, case):
    o = case['opts']
    return dbs_oracle.diverse_sample_beam(fam, fc, att, masks if case['masked'] else None, beam_size=case['beam_size'],
                                          group_size=case['group_size'], diversity_lambda=case['diversity_lambda'],
                                          sample_n=o.get('sample_n', 1), length_penalty=o.get('length_penalty', ''),
                                          temperature=o.get('temperature', 1.0), decoding_constraint=bool(o.get('decoding_constraint', 0)))


@pytest.mark.parametrize('family', ['updown', 'aoa'])
def test_restatement_reproduces_reference(family):
    g, cases, meta = _small()
    W, fc, att, masks, dims = small_setup(family, g, meta)
    fam = co.Family(family, W, dims[-1], heads=AOA_HEADS)
    for case in cases:
        key = '%s_%s_' % (family, case['name'])
        seq, lp, done = oracle_case(fam, fc, att, masks, case)
        assert np.array_equal(seq.numpy(), g[key + 'seq']), case['name']
        picked = lp.gather(2, seq.unsqueeze(2)).squeeze(2)
        assert np.abs(picked.numpy() - g[key + 'picked']).max() < 1e-5, case['name']
        dseq, dlen, dp = dbs_oracle.beams_to_arrays(done, case['beam_size'], dims[-1])
        assert np.array_equal(dseq, g[key + 'done_seq']) and np.array_equal(dlen, g[key + 'done_len']), case['name']
        assert np.abs(dp - g[key + 'done_p']).max() < 1e-4, case['name']
        for j, rec in enumerate(done[0]):
            L = rec['logps'].shape[0]
            np.testing.assert_allclose(rec['logps'].numpy(), g[key + 'logps0'][j, :L], rtol=0, atol=1e-5, err_msg='%s %d' % (case['name'], j))


def test_restatement_group_order_and_padding():
    """done_beams is group-concatenated (each group sorted, not the whole list); with sample_n == bdash only the first B rows are filled."""
    g, cases, meta = _small()
    W, fc, att, masks, dims = small_setup('updown', g, meta)
    fam = co.Family('updown', W, dims[-1])
    seq, lp, done = dbs_oracle.diverse_sample_beam(fam, fc, att, beam_size=6, group_size=3, diversity_lambda=2.0, sample_n=2)
    B = fc.shape[0]
    assert seq.shape[0] == 2 * B and not seq[B:].any() and not lp[B:].any()
    for recs in done:
        ps = [r['p'] for r in recs]
        for grp in range(3):
            assert ps[2 * grp] >= ps[2 * grp + 1]


def test_diverse_guards():
    """Diverse beam search configurations the engine does not run raise before any device work."""
    import imagecaptioning.pytorch_b200 as b200
    cfg = dict(V=30, E=16, H=16, A=8, F_fc=16, F_att=16, T=5)
    fc, att = co.make_inputs(2, 3, 16, 16, seed=1)
    updown = b200.setup(family_opt('updown', **cfg))
    for bad in ({'beam_size': 6, 'group_size': 4, 'sample_n': 1},                 # group_size does not divide beam_size
                {'beam_size': 6, 'group_size': 3, 'sample_n': 3},                 # sample_n not in {1, bdash}
                {'beam_size': 6, 'group_size': 3},                                # sample_n left at _sample_beam's default of 10
                {'beam_size': 6, 'group_size': 3, 'sample_n': 1, 'diversity_lambda': -0.5},
                {'beam_size': 1, 'group_size': 2},                                # _diverse_sample
                {'beam_size': 1, 'group_size': 2, 'sample_method': 'sample'}):
        with pytest.raises(NotImplementedError):
            updown(fc, att, None, opt=bad, mode='sample')
    newfc = b200.setup(make_opt('newfc', 60, 32, 32, 16, 48, 48, 8))
    fc2, att2 = torch.zeros(2, 48), torch.zeros(2, 3, 48)
    with pytest.raises(NotImplementedError, match='per core call'):
        newfc(fc2, att2, None, opt={'beam_size': 4, 'group_size': 2, 'sample_n': 1}, mode='sample')
    tfm = b200.setup(family_opt('transformer', 60, 32, 64, 2, 48, 48, 8, heads=4))
    with pytest.raises(NotImplementedError, match='one position per launch'):
        tfm(fc2, att2, None, opt={'beam_size': 4, 'group_size': 2, 'sample_n': 1}, mode='sample')


def test_diverse_options_reach_the_engine():
    """Valid diverse beam search options get past the guards and stop at the no-CPU-fallback check."""
    import imagecaptioning.pytorch_b200 as b200
    fc, att = torch.zeros(2, 48), torch.zeros(2, 3, 48)
    m = b200.setup(make_opt('updown', 60, 32, 32, 16, 48, 48, 8))
    aoa = b200.setup(family_opt('aoa', 60, 32, 32, 16, 48, 48, 8, heads=4))
    for ok in ({'beam_size': 4, 'group_size': 2, 'sample_n': 1}, {'beam_size': 6, 'group_size': 3, 'sample_n': 2, 'diversity_lambda': 2.0},
               {'beam_size': 4, 'group_size': 4, 'sample_n': 1, 'diversity_lambda': 0.0, 'decoding_constraint': 1, 'length_penalty': 'wu_0.5'},
               {'beam_size': 4, 'group_size': 2, 'sample_n': 1, 'temperature': 1.3}):
        for model in (m, aoa):
            with pytest.raises(RuntimeError, match='CUDA'):
                model(fc, att, None, opt=ok, mode='sample')


def test_diverse_abi_declared():
    """The two new entry points and the options struct are in the header and the ctypes table with matching layouts."""
    import ctypes
    from imagecaptioning.pytorch_b200 import _lib
    assert {'capb200_decode_beam_diverse', 'capb200_aoa_decode_beam_diverse'} <= set(_lib.SIGNATURES)
    assert ctypes.sizeof(_lib.DiverseOpts) == ctypes.sizeof(_lib.BeamOpts) + 8
    hdr = open(os.path.join(os.path.dirname(GOLD), '..', 'include', 'capb200.h')).read()
    assert 'capb200_diverse_opts' in hdr
