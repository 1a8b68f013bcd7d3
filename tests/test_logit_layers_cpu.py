"""logit_layers > 1 (AttModel's multi-layer output head, AttModel.py:87-92) on the CPU: the oracle's head against the live-reference golden
(tests/make_logit_layers_golden.py), reference checkpoints loading into the engine models, the Transformer ignoring the option, the
refusals, the head's place among the gradient groups, and the C ABI declarations of the head."""
import json
import os
import re

import numpy as np
import pytest
import torch

from helpers import REPO, co, family_opt
import logit_head_oracle as lho

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'logit_layers_small.npz')
FAMILIES = ('updown', 'att2in2', 'newfc', 'aoa')


def _golden():
    g = np.load(GOLD)
    return g, json.loads(str(g['meta'])), tuple(int(x) for x in g['cfg'])


def _weights(fam, meta, dims, dtype=torch.float32):
    V, E, H, A, F_fc, F_att, T = dims
    W = co.make_weights(fam, V, E, H, A, F_fc, F_att, seed=meta['seed'], logit_scale=meta['logit_scale'], logit_layers=meta['logit_layers'])
    fc, att = co.make_inputs(meta['B'], meta['R'], F_fc, F_att, seed=meta['seed'])
    return {k: v.to(dtype) for k, v in W.items()}, fc.to(dtype), att.to(dtype)


def _opt(fam, dims, k):
    V, E, H, A, F_fc, F_att, T = dims
    opt = family_opt(fam, V, E, H, A, F_fc, F_att, T, heads=4)
    opt.logit_layers = k
    return opt


@pytest.mark.parametrize('fam', FAMILIES)
def test_oracle_head_matches_reference_decode(fam):
    g, meta, dims = _golden()
    W, fc, att = _weights(fam, meta, dims)
    of = lho.family(fam, W, dims[-1], heads=4)
    p = fam + '_'
    seq, lp = co.sample(of, fc, att)
    assert np.array_equal(seq.numpy(), g[p + 'greedy_seq'])
    assert np.abs(lp.numpy() - g[p + 'greedy_lp']).max() < 1e-5
    bseq, _, done = co.sample_beam(of, fc, att, beam_size=meta['beam'], sample_n=1)
    assert np.array_equal(bseq.numpy(), g[p + 'beam_seq'])
    for i in range(meta['B']):
        for j, rec in enumerate(done[i]):
            L = rec['seq'].shape[0]
            assert np.array_equal(rec['seq'].numpy(), g[p + 'beam_done_seq'][i, j, :L])
            assert abs(float(rec['p']) - g[p + 'beam_done_p'][i, j]) < 1e-4
            assert np.abs(rec['logps'].numpy() - g[p + 'beam_done_logps'][i, j, :L]).max() < 1e-5
    labels = torch.from_numpy(g[p + 'tf_labels'])
    tf = co.forward_teacher(of, fc, att, labels[:, :-1].reshape(meta['B'], -1, labels.shape[1] - 1))
    assert np.abs(tf.numpy() - g[p + 'tf_lp']).max() < 1e-5


@pytest.mark.parametrize('fam', FAMILIES)
def test_oracle_head_xe_gradients_match_reference(fam):
    """Eval-mode XE loss and every parameter gradient, through the head, in float64 against the reference's fp32 autograd."""
    g, meta, dims = _golden()
    W, fc, att = _weights(fam, meta, dims, torch.float64)
    for t in W.values():
        t.requires_grad_(True)
    of = lho.family(fam, W, dims[-1], heads=4)
    p = fam + '_'
    labels, masks = torch.from_numpy(g[p + 'tf_labels']), torch.from_numpy(g[p + 'tf_masks']).double()
    lp = co.forward_teacher(of, fc, att, labels[:, :-1].reshape(meta['B'], -1, labels.shape[1] - 1)).reshape(labels.shape[0], -1, dims[0] + 1)
    loss = co.language_model_criterion(lp, labels[:, 1:], masks[:, 1:])
    loss.backward()
    assert abs(float(loss.detach()) - float(g[p + 'xe_loss'])) < 1e-5
    names = [k[len(p + 'grad_'):] for k in g.files if k.startswith(p + 'grad_')]
    assert sorted(names) == sorted(W), set(names) ^ set(W)
    assert any(n.startswith('logit.3.') for n in names)
    for n in names:
        ref = g[p + 'grad_' + n]
        mine = np.zeros(ref.shape) if W[n].grad is None else W[n].grad.numpy()
        assert np.abs(mine - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max()), (fam, n, np.abs(mine - ref).max())


@pytest.mark.parametrize('fam', FAMILIES)
def test_reference_checkpoint_loads_strict(fam):
    """The engine model's state_dict has the reference's names and shapes at k = 3, and a checkpoint of them loads with strict=True."""
    import imagecaptioning.pytorch_b200 as b200
    g, meta, dims = _golden()
    W, _, _ = _weights(fam, meta, dims)
    m = b200.setup(_opt(fam, dims, 3))
    assert {k: list(v.shape) for k, v in m.state_dict().items()} == meta['keys'][fam]
    m.load_state_dict(W, strict=True)
    assert isinstance(m.logit, torch.nn.Sequential) and len(m.logit) == 7
    assert [type(x).__name__ for x in m.logit] == ['Linear', 'ReLU', 'Dropout'] * 2 + ['Linear']
    assert all(m.logit[i].p == 0.5 for i in (2, 5))
    assert torch.equal(m._vocab_logit.weight, W['logit.6.weight'])
    assert [n for n, _ in m._head_named()] == ['logit.0.weight', 'logit.0.bias', 'logit.3.weight', 'logit.3.bias']


@pytest.mark.parametrize('fam', FAMILIES)
def test_single_layer_head_is_unchanged(fam):
    import imagecaptioning.pytorch_b200 as b200
    _, _, dims = _golden()
    m = b200.setup(_opt(fam, dims, 1))
    assert isinstance(m.logit, torch.nn.Linear) and m._head_named() == []
    assert 'logit.weight' in m.state_dict()


def test_transformer_ignores_logit_layers():
    import imagecaptioning.pytorch_b200 as b200
    opts = [family_opt('transformer', 60, 32, 64, 2, 48, 56, 8, heads=4) for _ in range(2)]
    opts[1].logit_layers = 3
    keys = [{k: tuple(v.shape) for k, v in b200.setup(o).state_dict().items()} for o in opts]
    assert keys[0] == keys[1]
    assert b200.setup(opts[1])._head_named() == []


@pytest.mark.parametrize('fam', FAMILIES + ('transformer',))
@pytest.mark.parametrize('k', [0, -1])
def test_nonpositive_logit_layers_refused(fam, k):
    import imagecaptioning.pytorch_b200 as b200
    opt = family_opt(fam, 60, 32, 32, 16, 48, 56, 8, heads=4)
    opt.logit_layers = k
    with pytest.raises(ValueError, match='logit_layers'):
        b200.setup(opt)


@pytest.mark.parametrize('fam', FAMILIES)
def test_use_bn_still_refused(fam):
    import imagecaptioning.pytorch_b200 as b200
    opt = _opt(fam, _golden()[2], 3)
    opt.use_bn = 1
    with pytest.raises(NotImplementedError, match='use_bn'):
        b200.setup(opt)


@pytest.mark.parametrize('fam', FAMILIES)
def test_head_gradients_join_group_zero(fam):
    """The head's hidden layers are trained with the model: their gradients sit in the flat buffer's group 0 with the vocabulary Linear's
    (the group the engine finishes first and a data-parallel caller all-reduces first)."""
    import imagecaptioning.pytorch_b200 as b200
    from imagecaptioning.pytorch_b200.models import _slot_name
    _, _, dims = _golden()
    m = b200.setup(_opt(fam, dims, 3))
    head = m._head_named()
    named = [(_slot_name(path), p) for path, p in m._grad_slots()] + head
    groups = m._grad_groups(named)
    assert [n for n, _ in groups[0]] == ['logit_w', 'logit_b'] + [n for n, _ in head]
    assert sum(len(g) for g in groups) == len(named)
    assert {id(p) for g in groups for _, p in g} == {id(p) for p in m.parameters()}


def _declaration(header, name):
    m = re.search(r'\b%s\s*\(([^;]*)\)\s*;' % name, header)
    assert m, name
    return [a.strip() for a in m.group(1).split(',')]


@pytest.mark.parametrize('abi', ['engine', 'aoa'])
def test_head_entry_points_declared_and_typed(abi):
    """include/capb200.h and _lib.SIGNATURES agree on the head's entry points: the same argument count, pointer arrays as pointers."""
    import ctypes
    from imagecaptioning.pytorch_b200 import _lib
    header = open(os.path.join(REPO, 'include', 'capb200.h')).read()
    handle = 'capb200_engine*' if abi == 'engine' else 'capb200_aoa_engine*'
    grad_args = _declaration(header, 'capb200_%s_bind_logit_head_grads' % abi)
    drop_args = _declaration(header, 'capb200_%s_set_logit_dropout' % abi)
    assert [a.split()[-1] for a in grad_args[1:]] == ['gw', 'gb'] and drop_args[1] == 'float p'
    res, args = _lib.SIGNATURES['capb200_%s_bind_logit_head_grads' % abi]
    assert len(args) == len(grad_args) and args[1] == args[2] == ctypes.POINTER(ctypes.c_void_p)
    assert _lib.SIGNATURES['capb200_%s_set_logit_dropout' % abi][1] == [ctypes.c_void_p, ctypes.c_float]
    set_args = _declaration(header, 'capb200_%s_set_logit_layers' % abi)
    bind_args = _declaration(header, 'capb200_%s_bind_logit_head' % abi)
    assert set_args[0].replace(' ', '').startswith(handle) and set_args[1] == 'int logit_layers'
    assert bind_args[0].replace(' ', '').startswith(handle)
    assert [a.split()[-1] for a in bind_args[1:]] == ['w', 'b', 'stream'] and all('const float* const*' in a for a in bind_args[1:3])
    res, args = _lib.SIGNATURES['capb200_%s_set_logit_layers' % abi]
    assert res is ctypes.c_int and args == [ctypes.c_void_p, ctypes.c_int]
    res, args = _lib.SIGNATURES['capb200_%s_bind_logit_head' % abi]
    assert res is ctypes.c_int and len(args) == len(bind_args) and args[1] == args[2] == ctypes.POINTER(ctypes.c_void_p)
