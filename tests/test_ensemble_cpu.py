"""Test-time ensembles without a GPU: the restatement in ensemble_oracle against the reference's AttEnsemble goldens, and every refusal of
the Python mirror and the C ABI, which must come before any device work."""
import ctypes
import itertools
import json
import os

import numpy as np
import pytest
import torch

from helpers import co, family_opt
import dbs_oracle
import ensemble_oracle as eo

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ensemble_small.npz')


def _golden():
    g = np.load(GOLD)
    return g, json.loads(str(g['meta']))


def assert_rows_close(mine, ref, atol, what):
    """Equal -inf pattern (a mixture that underflows, or a decode edit) and finite entries within atol."""
    mine, ref = np.asarray(mine), np.asarray(ref)
    assert np.array_equal(np.isneginf(mine), np.isneginf(ref)), what
    fin = np.isfinite(ref)
    assert np.abs(mine[fin] - ref[fin]).max(initial=0.0) < atol, (what, float(np.abs(mine[fin] - ref[fin]).max(initial=0.0)))


def test_restatement_reproduces_reference():
    g, meta = _golden()
    c = meta['cfg']
    fc, att = co.make_inputs(meta['B'], meta['R'], c['F_fc'], c['F_att'], seed=meta['input_seed'])
    n = 0
    for mix, wname, (name, opts, masked) in itertools.product(meta['mixes'], meta['weights'], meta['cases']):
        key = '%s_%s_%s_' % (mix, wname, name)
        out = eo.run_oracle(eo.oracle_for(meta, mix, wname), fc, att, meta, opts, masked)
        if opts == 'teacher':
            assert_rows_close(out['out'].numpy(), g[key + 'out'], 1e-5, key)
            n += 1
            continue
        assert np.array_equal(out['seq'].numpy(), g[key + 'seq']), key
        assert_rows_close(out['logprobs'].numpy(), g[key + 'logprobs'], 1e-5, key)
        if 'done' in out:
            dseq, dlen, dp = dbs_oracle.beams_to_arrays(out['done'], opts['beam_size'], c['T'])
            assert np.array_equal(dseq, g[key + 'done_seq']) and np.array_equal(dlen, g[key + 'done_len']), key
            assert np.abs(dp - g[key + 'done_p']).max() < 1e-4, key
        n += 1
    assert n == 3 * 2 * 4


def test_one_member_is_the_single_model():
    """A one-member ensemble mixes softmax(z) * w / w back into the member's own log-probs."""
    g, meta = _golden()
    c = meta['cfg']
    fc, att = co.make_inputs(meta['B'], meta['R'], c['F_fc'], c['F_att'], seed=meta['input_seed'])
    (f, W), = eo.member_weight_dicts(meta, 'updown2')[:1]
    single = eo.member_family(f, W, c['T'])
    seq, lp = co.sample(single, fc, att)
    eseq, elp = co.sample(eo.EnsembleFamily([single], [3.0]), fc, att)
    assert torch.equal(seq, eseq) and float((lp - elp).abs().max()) < 1e-5


def _members(V=30, T=5, **kw):
    import imagecaptioning.pytorch_b200 as b200
    return [b200.setup(family_opt(f, V, 16, 16, 8, 16, 16, T, heads=4)) for f in ('updown', 'att2in2', 'newfc', 'aoa')]


def test_python_refusals():
    """Everything AttEnsemble cannot mean on the engine raises NotImplementedError or ValueError before any device work (on this box the
    first device work would raise RuntimeError: no CUDA)."""
    import imagecaptioning.pytorch_b200 as b200
    ups, att2, newfc, aoa = _members()
    E = b200.B200AttEnsemble
    with pytest.raises(ValueError):
        E([])
    with pytest.raises(ValueError):
        E([ups] * 9)
    with pytest.raises(NotImplementedError):
        E([ups, b200.setup(family_opt('transformer', 30, 16, 32, 1, 16, 16, 5, heads=4))])
    with pytest.raises(ValueError, match='vocab_size'):
        E([ups, b200.setup(family_opt('updown', 31, 16, 16, 8, 16, 16, 5))])
    with pytest.raises(ValueError, match='seq_length'):
        E([ups, b200.setup(family_opt('updown', 30, 16, 16, 8, 16, 16, 6))])
    for bad in ([1.0, -1.0], [0.0, 0.0], [1.0, float('nan')], [1.0, float('inf')], [1.0]):
        with pytest.raises(ValueError):
            E([ups, aoa], weights=bad)
    ens = E([ups, att2, newfc, aoa], weights=[1.0, 2.0, 0.5, 1.0])
    fc, att = torch.zeros(2, 16), torch.zeros(2, 3, 16)
    with pytest.raises(NotImplementedError):
        ens(fc, att, None, opt={'beam_size': 4, 'group_size': 2, 'sample_n': 1}, mode='sample')
    with pytest.raises(NotImplementedError):
        ens(fc, att, None, opt={'beam_size': 1, 'group_size': 2}, mode='sample')
    with pytest.raises(NotImplementedError):
        ens(fc, att, None, opt={'beam_size': 1, 'output_logsoftmax': 0}, mode='sample')
    with pytest.raises(NotImplementedError):
        ens.scst_step(fc, att, None, None, 5)
    with pytest.raises(NotImplementedError):
        ens.xe_step(fc, att, None, None)
    ens.seq_length = 7                          # eval_ensemble.py sets model.seq_length; the members decode their own max_length
    with pytest.raises(ValueError, match='max_length'):
        ens(fc, att, None, opt={'beam_size': 3, 'sample_n': 1}, mode='sample')
    ens.seq_length = ups.seq_length
    ens.weights.fill_(0.0)                      # a weights buffer edited after construction is checked at the call
    with pytest.raises(ValueError):
        ens(fc, att, None, opt={'beam_size': 3, 'sample_n': 1}, mode='sample')
    split = E([ups, b200.setup(family_opt('updown', 30, 16, 16, 8, 16, 16, 5)).to('meta')])
    with pytest.raises(ValueError, match='device'):
        split(fc, att, None, opt={'beam_size': 3, 'sample_n': 1}, mode='sample')


def test_python_mirror_surface():
    """Reference attributes: vocab_size / seq_length / bad_endings_ix from models[0], the weights buffer and the state_dict layout."""
    import imagecaptioning.pytorch_b200 as b200
    ups, att2, newfc, aoa = _members()
    ens = b200.B200AttEnsemble([ups, newfc])
    assert (ens.vocab_size, ens.seq_length, ens.bad_endings_ix) == (ups.vocab_size, ups.seq_length, ups.bad_endings_ix)
    assert ens.weights.dtype == torch.float32 and ens.weights.tolist() == [1.0, 1.0]
    keys = set(ens.state_dict())
    assert 'weights' in keys and {'models.0.' + k for k in ups.state_dict()} <= keys and {'models.1.' + k for k in newfc.state_dict()} <= keys
    with pytest.raises(RuntimeError, match='CUDA'):           # valid options reach the no-CPU-fallback check
        ens(torch.zeros(2, 16), torch.zeros(2, 3, 16), None, opt={'beam_size': 3, 'sample_n': 1, 'length_penalty': 'wu_0.5'}, mode='sample')


@pytest.fixture(scope='module')
def lib():
    import __graft_entry__ as ge
    ge.build()
    import imagecaptioning.pytorch_b200 as b200
    return b200._lib.load()


def test_cabi_refusals(lib):
    """The C entry points refuse K outside 1..8, null or unknown members and bad weight vectors before touching any engine or the device."""
    from imagecaptioning.pytorch_b200 import _lib
    s = lib.capb200_ensemble_create()
    assert s
    fake = ctypes.c_void_p(0x1000)              # never dereferenced: every refusal below comes first
    seq = ctypes.c_void_p(0x2000)

    def call(members, K):
        bo = _lib.BeamOpts(3, 1)
        so = _lib.SampleOpts(1, _lib.SAMPLE_GREEDY)
        rb = lib.capb200_ensemble_decode_beam(s, members, K, None, None, None, 2, 3, ctypes.byref(bo), seq, None, None, None, None, None, None)
        rs = lib.capb200_ensemble_decode_sample(s, members, K, None, None, None, 2, 3, ctypes.byref(so), None, 0, seq, seq, None, None)
        return rb, rs

    def members(*spec):
        arr = (_lib.EnsembleMember * len(spec))()
        for k, (fam, eng, w) in enumerate(spec):
            arr[k].family, arr[k].engine, arr[k].weight = fam, eng, w
        return arr

    ok = members((_lib.FAMILY_UPDOWN, fake, 1.0))
    assert call(ok, 0) == (1, 1) and b'1..8' in lib.capb200_last_error()
    assert call(members(*[(_lib.FAMILY_UPDOWN, fake, 1.0)] * 9), 9) == (1, 1) and b'1..8' in lib.capb200_last_error()
    assert call(None, 2) == (1, 1)
    for spec, msg in ((((0, fake, 1.0), (0, fake, -1.0)), b'>= 0'), (((0, fake, 0.0), (3, fake, 0.0)), b'all be zero'),
                      (((0, fake, float('nan')),), b'finite'), (((0, None, 1.0),), b'null member'), (((7, fake, 1.0),), b'AoANet')):
        assert call(members(*spec), len(spec)) == (1, 1), spec
        assert msg in lib.capb200_last_error(), (spec, lib.capb200_last_error())
    assert lib.capb200_ensemble_launch_count(s) == 0
    lib.capb200_ensemble_destroy(s)
