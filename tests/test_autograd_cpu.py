"""CPU checks of the autograd path (model.autograd): the opt plumbing, the C ABI of the *_vjp entry points, and the refusals it adds --
raised before any device work with the flag on, while the same call with the flag off still stops at the no-CPU-fallback RuntimeError."""
import ctypes
import os
import re

import pytest
import torch

from helpers import REPO, family_opt

FAMILIES = {'updown': 'updown', 'att2in2': 'att2in2', 'newfc': 'newfc', 'aoa': 'aoa', 'transformer': 'tfm'}


def _model(family, flag):
    import imagecaptioning.pytorch_b200 as b200
    A = 2 if family == 'transformer' else (0 if family == 'aoa' else 16)
    opt = family_opt(family, 60, 32, 32, A, 48, 48, 8, heads=4)
    if flag is not None:
        opt.b200_autograd = flag
    return b200.setup(opt)


@pytest.mark.parametrize('family', sorted(FAMILIES))
def test_flag_plumbing(family):
    assert _model(family, None).autograd is False
    assert _model(family, 0).autograd is False
    m = _model(family, 1)
    assert m.autograd is True and m._autograd_active()
    with torch.no_grad():
        assert not m._autograd_active()
    for p in m.parameters():
        p.requires_grad_(False)
    assert not m._autograd_active()
    m.autograd = False
    for p in m.parameters():
        p.requires_grad_(True)
    assert not m._autograd_active()


def test_vjp_entry_points_in_header_and_signatures():
    import imagecaptioning.pytorch_b200 as b200
    L = b200._lib
    header = open(os.path.join(REPO, 'include', 'capb200.h')).read()
    declared = set(re.findall(r'\b(capb200_[a-z0-9]+_(?:xe|scst)_vjp)\s*\(', header))
    want = {'capb200_%s_%s_vjp' % (p, k) for p in FAMILIES.values() for k in ('xe', 'scst')}
    assert declared == want
    assert want <= set(L.SIGNATURES)
    # capb200_vjp_opts { int forward_only; const float* dlogprobs; int greedy; }: the ctypes mirror has the C layout
    body = header.split('} capb200_vjp_opts;')[0].rsplit('typedef struct {', 1)[1]
    fields = re.findall(r'^\s*(?:const )?(\w+\*?)\s+(\w+);', body, re.M)
    assert [n for _, n in fields] == [n for n, _ in L.VjpOpts._fields_]
    assert ctypes.sizeof(L.VjpOpts) == 24 and L.VjpOpts.dlogprobs.offset == 8 and L.VjpOpts.greedy.offset == 16
    # each entry takes the family's option struct, then the vjp options, then (xe) labels / label_cols or (scst) the gradient table
    for fam, prefix in FAMILIES.items():
        opts = {'updown': L.XeOpts, 'att2in2': L.XeOpts, 'newfc': L.XeOpts, 'aoa': L.AoaXeOpts, 'transformer': L.TfmXeOpts}[fam]
        _, xe_args = L.SIGNATURES['capb200_%s_xe_vjp' % prefix]
        _, sc_args = L.SIGNATURES['capb200_%s_scst_vjp' % prefix]
        i = xe_args.index(ctypes.POINTER(opts))
        assert xe_args[i + 1] is ctypes.POINTER(L.VjpOpts) and sc_args[i + 1] is ctypes.POINTER(L.VjpOpts)
        assert len(xe_args) == i + 7 and len(sc_args) == i + 6


def _feats(family):
    fc, att = torch.zeros(2, 48), torch.zeros(2, 3, 48)
    labels = torch.zeros(2, 9, dtype=torch.long)
    labels[:, 1:4] = 5
    return fc, att, labels


REFUSED = [{'beam_size': 3, 'sample_n': 1}, {'sample_method': 'top5'}, {'sample_method': 'top0.9'}, {'sample_method': 'gumbel'}, {'decoding_constraint': 1},
           {'remove_bad_endings': 1}, {'suppress_UNK': 1}, {'block_trigrams': 1}]


@pytest.mark.parametrize('family', sorted(FAMILIES))
def test_refusals_with_flag_on_only(family):
    fc, att, labels = _feats(family)
    for flag in (1, 0):
        m = _model(family, flag).train()
        for opt in REFUSED:
            if flag:
                with pytest.raises(NotImplementedError):
                    m(fc, att, None, opt=dict(opt), mode='sample')
            else:
                with pytest.raises(RuntimeError, match='CUDA'):
                    m(fc, att, None, opt=dict(opt), mode='sample')
        # features that require grad
        for f, a in ((fc.clone().requires_grad_(), att), (fc, att.clone().requires_grad_())):
            if flag:
                with pytest.raises(NotImplementedError):
                    m(f, a, None, opt={'sample_method': 'sample'}, mode='sample')
                with pytest.raises(NotImplementedError):
                    m(f, a, labels)
            else:
                with pytest.raises(RuntimeError, match='CUDA'):
                    m(f, a, labels)
        # covered calls get past the guards and stop at the device
        for opt in ({'sample_method': 'greedy'}, {'sample_method': 'sample', 'sample_n': 3, 'temperature': 0.7}):
            with pytest.raises(RuntimeError, match='CUDA'):
                m(fc, att, None, opt=opt, mode='sample')
        with pytest.raises(RuntimeError, match='CUDA'):
            m(fc, att, labels)


def test_eval_mode_truncated_samplers_pass_the_guards():
    """top-k / top-p / gumbel are refused in train mode only: in eval mode the decode path draws and the autograd forward replays."""
    fc, att, _ = _feats('updown')
    m = _model('updown', 1).eval()
    for method in ('top5', 'top0.9', 'gumbel'):
        with pytest.raises(RuntimeError, match='CUDA'):
            m(fc, att, None, opt={'sample_method': method}, mode='sample')


def test_scheduled_sampling_refusal_unchanged_with_flag_off():
    fc, att, labels = _feats('updown')
    m = _model('updown', 0).train()
    m.ss_prob = 0.25
    with pytest.raises(NotImplementedError, match='scheduled sampling'):
        m(fc, att, labels)
    m.autograd = True
    with pytest.raises(RuntimeError, match='CUDA'):
        m(fc, att, labels)
