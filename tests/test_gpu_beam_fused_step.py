"""GPU: UpDown beam search with each step's vocabulary statistics / top-k, beam step and next-step state gather fused into one kernel per
image (beam_search_step_kernel) against the separate kernels, through capb200_decode_beam_form: seq, the log-prob rows and done_beams
(sequences, lengths, scores) must be bitwise equal, over eager, captured and replayed calls, and each fused decode must issue exactly
2T - 1 fewer launches.  Cases the fused kernel does not cover must run the separate kernels under the automatic form."""
import ctypes

import pytest
import torch

from imagecaptioning.pytorch_b200 import _lib
from imagecaptioning.pytorch_b200 import synthetic as syn

pytestmark = pytest.mark.gpu

SMALL = dict(V=511, E=64, H=64, A=32, F_fc=48, F_att=48)        # V + 1 = 512 and H = 64: 16-byte aligned rows
R = 9


def _model(T, eos_bias=0.0, cfg=SMALL, logit_scale=8.0):
    model = syn.build_model('updown', T=T, seed=41, logit_scale=logit_scale, mode='tc_f16x3', **cfg)
    if eos_bias:
        with torch.no_grad():
            model.logit.bias[0] += eos_bias            # makes <eos> a frequent candidate: records are appended mid-loop
    return model


def _inputs(B, cfg=SMALL, masked=False):
    fc, att = syn.make_inputs(B, R, cfg['F_fc'], cfg['F_att'], seed=7 + B)
    masks = None
    if masked:
        n = torch.randint(1, R + 1, (B,), generator=torch.Generator().manual_seed(B))
        n[0] = R                                        # the batch keeps all R columns after the model's clip
        masks = (torch.arange(R)[None, :] < n[:, None]).float().cuda()
    return fc.cuda(), att.cuda(), masks


def _decode(model, form, fc, att, masks, opt):
    """One beam decode through capb200_decode_beam_form; returns the outputs (copies) and the launches it issued."""
    def call(lib, fc_, att_, masks_, B, R_, bo, seq, logprobs, d_seq, d_len, d_p, d_raw):
        return lib.capb200_decode_beam_form(form, model._engine, _lib.ptr(fc_), _lib.ptr(att_), _lib.ptr(masks_), B, R_, ctypes.byref(bo),
                                            _lib.ptr(seq), _lib.ptr(logprobs), _lib.ptr(d_seq), _lib.ptr(d_len), _lib.ptr(d_p), _lib.ptr(d_raw),
                                            _lib.current_stream())
    model._call_beam = call
    try:
        l0 = model.launch_count
        with torch.no_grad():     # _sample_beam directly: the model's sample mode runs greedy decoding at beam size 1
            seq, lp = model._sample_beam(fc, att, masks, opt=opt)
        torch.cuda.synchronize()
        launches = model.launch_count - l0
    finally:
        del model._call_beam
    d_seq, d_len, d_p, d_raw = model._last_beam
    return [t.clone() for t in (seq, lp, d_seq, d_len, d_p, d_raw)], launches


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _same(a, b):
    for x, y, name in zip(a, b, ('seq', 'seq_logprobs', 'done_seq', 'done_len', 'done_p', 'done_raw')):
        assert torch.equal(_bits(x), _bits(y)), name


def _compare(model, fc, att, masks, opt, T, calls=3):
    """`calls` decodes per form (eager, captured, replayed): every call of the fused form equals the separate kernels' bitwise.  The
    model's first call also binds its weights, so launch counts are compared from each form's second call on, and the eager call of
    each form must count what its captured call counts."""
    ref = [_decode(model, 1, fc, att, masks, opt) for _ in range(calls)]
    fused = [_decode(model, 2, fc, att, masks, opt) for _ in range(calls)]
    auto = _decode(model, 0, fc, att, masks, opt)
    for (r, _), (f, _) in zip(ref, fused):
        _same(r, f)
    _same(ref[0][0], auto[0])
    lr, lf = [n for _, n in ref], [n for _, n in fused]
    assert len(set(lr[1:])) == 1 and len(set(lf)) == 1, (lr, lf)
    assert lr[1] - lf[1] == 2 * T - 1, (lr, lf)
    assert auto[1] == lf[1]                             # the automatic form picks the fused kernel
    return ref[0][0]


@pytest.mark.parametrize('T', [1, 20, 64])
@pytest.mark.parametrize('beam', [1, 2, 5, 10, 16])
@pytest.mark.parametrize('B', [1, 7, 256])
def test_fused_step_matches_separate_kernels(B, beam, T):
    model = _model(T)
    fc, att, masks = _inputs(B)
    _compare(model, fc, att, masks, {'beam_size': beam, 'sample_n': 1}, T)


@pytest.mark.parametrize('beam', [2, 5, 16])
def test_fused_step_masks_penalty_and_eos(beam):
    T = 20
    model = _model(T, eos_bias=4.0)
    fc, att, masks = _inputs(7, masked=True)
    out = _compare(model, fc, att, masks, {'beam_size': beam, 'sample_n': beam, 'length_penalty': 'wu_0.5'}, T)
    lens = out[3].cpu().numpy()
    assert (lens < T).any(), 'the EOS-heavy model should finish beams before the last step'


def test_fused_step_headline_shape():
    """The bench.py shape: V + 1 = 9488, E = H = 1000, 36 regions, beam 5, T 20, 256 images."""
    import bench
    cfg = {k: bench.CFG[k] for k in ('V', 'E', 'H', 'A', 'F_fc', 'F_att')}
    model = _model(bench.CFG['T'], cfg=cfg, logit_scale=12.0)
    fc, att = syn.make_inputs(256, bench.R, cfg['F_fc'], cfg['F_att'], seed=1234)
    _compare(model, fc.cuda(), att.cuda(), None, {'beam_size': 5, 'sample_n': 1}, bench.CFG['T'], calls=2)


@pytest.mark.parametrize('opt', [{'decoding_constraint': 1}, {'temperature': 1.3}])
def test_uncovered_options_keep_the_separate_kernels(opt):
    T = 20
    model = _model(T)
    fc, att, masks = _inputs(7)
    opt = dict(opt, beam_size=5, sample_n=1)
    _decode(model, 1, fc, att, masks, dict(opt, beam_size=4))     # binds the weights (launches of their own) under another graph key
    ref, lr = _decode(model, 1, fc, att, masks, opt)
    auto, la = _decode(model, 0, fc, att, masks, opt)
    _same(ref, auto)
    assert la == lr
    with pytest.raises(RuntimeError, match='fused beam step'):
        _decode(model, 2, fc, att, masks, opt)
