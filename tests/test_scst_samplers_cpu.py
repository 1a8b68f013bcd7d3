"""CPU checks of the selectable self-critical samplers: the C header and the ctypes mirrors agree (the sampler pointer sits just before
reward_weights, which stays last), the reference's sample_method names map to the engine's methods, B200LossWrapper hands
train_sample_method / sc_sample_method to the fused steps (and nothing extra for the defaults), and what stays out of scope is refused
before any device work."""
import argparse
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from helpers import co, family_opt

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_sampler_struct_mirrors_header():
    import imagecaptioning.pytorch_b200 as b200
    L = b200._lib
    hdr = open(os.path.join(REPO, 'include', 'capb200.h')).read()
    body = re.sub(r'/\*.*?\*/', '', re.search(r'typedef struct \{([^{}]*)\} capb200_sampler_opts;', hdr).group(1), flags=re.S)
    fields = [f for decl in body.split(';') if decl.strip() for f in re.findall(r'(\w+)\s*(?:,|$)', decl.strip())]
    assert fields == [f for f, _ in L.SamplerOpts._fields_]
    assert [t for _, t in L.SamplerOpts._fields_] == [ctypes.c_int, ctypes.c_float, ctypes.c_int, ctypes.c_float, ctypes.c_void_p]
    for py in (L.ScstOpts, L.AoaScstOpts, L.TfmScstOpts):
        assert py._fields_[-2] == ('sampler', ctypes.POINTER(L.SamplerOpts))
        assert py._fields_[-1] == ('reward_weights', ctypes.POINTER(L.RewardWeights))
        assert not py().sampler                         # zero-initialised: NULL, the multinomial samples and the greedy baseline
    for name in ('GREEDY', 'MULTINOMIAL', 'TOPK', 'TOPP'):
        assert int(re.search(r'#define CAPB200_SAMPLE_%s (\d+)' % name, hdr).group(1)) == getattr(L, 'SAMPLE_' + name)


def test_sampling_method_names():
    import imagecaptioning.pytorch_b200 as b200
    L, sm = b200._lib, b200.models.sampling_method
    assert sm('greedy') == (L.SAMPLE_GREEDY, 0.0, False)
    assert sm('sample') == (L.SAMPLE_MULTINOMIAL, 0.0, False)
    assert sm('gumbel') == (L.SAMPLE_MULTINOMIAL, 0.0, True)
    assert sm('top5') == (L.SAMPLE_TOPK, 5.0, False)
    assert sm('top0.9') == (L.SAMPLE_TOPP, 0.9, False)
    assert sm('top1') == (L.SAMPLE_TOPK, 1.0, False)
    for bad in ('top0', 'top-2'):
        with pytest.raises(ValueError):
            sm(bad)
    for bad in ('beam_search', 'dbs', 'topk'):
        with pytest.raises((NotImplementedError, ValueError)):
            sm(bad)


def test_scst_sampler_struct():
    import imagecaptioning.pytorch_b200 as b200
    L, make = b200._lib, b200.models._scst_sampler
    assert make('sample', 'greedy', None, False, 2, 5, 11, 0.7, 'cpu') == (None, None, 0.7)       # the default passes no struct
    ptr, keep, temp = make('gumbel', 'top0.5', None, False, 2, 5, 11, 0.7, 'cpu')
    s = ptr.contents
    assert (s.train_method, s.baseline_method, temp) == (L.SAMPLE_MULTINOMIAL, L.SAMPLE_TOPP, 1.0)      # gumbel: temperature 1
    assert abs(s.baseline_top - 0.5) < 1e-7 and not s.forced_baseline
    fb = torch.ones(2, 5, dtype=torch.long)
    ptr, keep, _ = make('top3', 'greedy', fb, False, 2, 5, 11, 1.0, 'cpu')
    assert ptr.contents.train_method == L.SAMPLE_TOPK and ptr.contents.forced_baseline == keep[1].data_ptr()
    with pytest.raises(ValueError, match='leave-one-out'):
        make('sample', 'top3', None, True, 2, 5, 11, 1.0, 'cpu')
    with pytest.raises(ValueError, match='leave-one-out'):
        make('sample', 'greedy', fb, True, 2, 5, 11, 1.0, 'cpu')
    with pytest.raises(ValueError, match='vocab_size'):
        make('top12', 'greedy', None, False, 2, 5, 11, 1.0, 'cpu')


def _wrapper(calls, **over):
    import imagecaptioning.pytorch_b200 as b200
    model = b200.setup(family_opt('updown', 30, 16, 16, 8, 16, 16, 5))
    opt = dict(sc_sample_method='greedy', sc_beam_size=1, train_sample_method='sample', train_beam_size=1, train_sample_n=2,
               cider_reward_weight=1, bleu_reward_weight=0, label_smoothing=0.0, structure_loss_weight=1.0,
               structure_loss_type='new_self_critical', use_ppo=0)
    opt.update(over)

    def fake_step(*args, **kwargs):
        calls.append(kwargs)
        raise RuntimeError('stop before the device')
    model.scst_step = fake_step
    b200.rewards.reset_scorer()
    b200.rewards.CiderD_scorer = object()
    return b200.B200LossWrapper(model, argparse.Namespace(**opt))


@pytest.mark.parametrize('train,base', [('sample', 'greedy'), ('top5', 'greedy'), ('greedy', 'top0.9'), ('gumbel', 'sample'), ('top0.5', 'top3')])
def test_loss_wrapper_hands_samplers_to_the_fused_step(train, base):
    import imagecaptioning.pytorch_b200 as b200
    fc, att = co.make_inputs(2, 3, 16, 16, seed=1)
    gts = [np.zeros((5, 7), np.int64)] * 2
    try:
        for sc, struc in ((True, False), (False, True)):
            calls = []
            lw = _wrapper(calls, train_sample_method=train, sc_sample_method=base)
            with pytest.raises(RuntimeError, match='stop before'):
                lw(fc, att, None, None, None, gts, torch.arange(2), sc, struc, False)
            kw = calls[0]
            assert kw.get('sample_method', 'sample') == train
            # new_self_critical has no baseline captions: sc_sample_method is not read there (loss_wrapper.py:25-53)
            assert kw.get('baseline_method', 'greedy') == (base if sc else 'greedy')
            if train == 'sample':
                assert 'sample_method' not in kw
            if base == 'greedy' or not sc:
                assert 'baseline_method' not in kw
    finally:
        b200.rewards.reset_scorer()


@pytest.mark.parametrize('over', [dict(sc_beam_size=2), dict(train_beam_size=2), dict(sc_sample_method='beam_search'),
                                  dict(train_sample_method='dbs'), dict(train_sample_method='top0')])
def test_out_of_scope_settings_still_refused(over):
    import imagecaptioning.pytorch_b200 as b200
    calls = []
    lw = _wrapper(calls, **over)
    fc, att = co.make_inputs(2, 3, 16, 16, seed=1)
    gts = [np.zeros((5, 7), np.int64)] * 2
    try:
        with pytest.raises(NotImplementedError):
            lw(fc, att, None, None, None, gts, torch.arange(2), True, False, False)
        assert calls == []
    finally:
        b200.rewards.reset_scorer()


def test_scst_step_refuses_bad_samplers_before_device_work():
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    fc, att = co.make_inputs(2, 3, 16, 16, seed=1)
    gts = cdo.make_refs(2, 30, seed=2)
    for family in ('updown', 'aoa', 'transformer'):
        m = b200.setup(family_opt(family, 30, 16, 32, 2 if family == 'transformer' else 8, 16, 16, 5, heads=4))
        for kw, exc in ((dict(sample_method='beam_search'), NotImplementedError), (dict(baseline_method='top0'), ValueError),
                        (dict(baseline='leave_one_out', baseline_method='top3'), ValueError), (dict(sample_method='top99'), ValueError)):
            with pytest.raises(exc):
                m.scst_step(fc, att, gts, None, 2, **kw)
