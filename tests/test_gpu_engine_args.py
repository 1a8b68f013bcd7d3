"""The decode entry points of every engine and of the ensemble check their options the same way: the same invalid options are refused with
the same message, before any kernel is launched."""
import ctypes
import re

import pytest
import torch

from helpers import co, family_opt
from imagecaptioning.pytorch_b200 import _lib

pytestmark = pytest.mark.gpu

CFG = dict(V=60, E=32, H=32, A=16, F_fc=48, F_att=48, T=8)
TFM_CFG = dict(V=60, E=32, H=64, A=2, F_fc=48, F_att=48, T=8)      # E = d_model, H = d_ff, A = layers per stack
B, R = 2, 5


def engine_model(family, c):
    import imagecaptioning.pytorch_b200 as b200
    dims = (c['V'], c['E'], c['H'], c['A'], c['F_fc'], c['F_att'])
    m = b200.setup(family_opt(family, *dims, c['T'], heads=4), numeric_mode='tc_f16x3')
    m.load_state_dict(co.make_weights(family, *dims, seed=3, logit_scale=5.0), strict=True)
    return m.cuda().eval()


def models():
    import imagecaptioning.pytorch_b200 as b200
    out = {f: engine_model(f, CFG) for f in ('updown', 'att2in2', 'newfc', 'aoa')}
    out['transformer'] = engine_model('transformer', TFM_CFG)
    out['ensemble'] = b200.B200AttEnsemble([out['updown'], out['aoa']], weights=[1.0, 2.0])
    return out


def refused(model, call):
    """Runs `call(lib)` on the model's engine; returns the error message of its refusal (without the checked condition), asserting that the
    call failed and launched nothing."""
    lib = model._ensure_engine(torch.device('cuda', torch.cuda.current_device()))
    before = model.launch_count
    rc = call(lib)
    torch.cuda.synchronize()
    assert rc != 0
    assert model.launch_count == before
    return lib.capb200_last_error().decode().split(' -- ', 1)[1]


def test_engines_refuse_the_same_options_alike():
    ms = models()
    fc, att = (x.cuda() for x in co.make_inputs(B, R, CFG['F_fc'], CFG['F_att'], seed=1))
    T, V1 = CFG['T'], CFG['V'] + 1
    seq = torch.zeros(B * 17, T + 2, dtype=torch.long, device='cuda')
    lp = torch.zeros(B * 17, T + 2, V1, device='cuda')
    done = [torch.zeros(B * 17 * T, dtype=dt, device='cuda') for dt in (torch.long, torch.int32, torch.float32, torch.float32)]
    tok = torch.zeros(B, T, dtype=torch.long, device='cuda')

    def sample(so, ld_tok=0, tokens=None):
        return lambda m: (lambda lib: m._call_sample(lib, fc, att, None, B, R, so, tokens, ld_tok, seq, lp))

    def beam(bo):
        return lambda m: (lambda lib: m._call_beam(lib, fc, att, None, B, R, bo, seq, lp, *done))

    cases = {
        'top-k at temperature 0': (sample(_lib.SampleOpts(1, _lib.SAMPLE_TOPK, temperature=0.0, top=3.0)), 'temperature must be positive'),
        'nucleus at temperature 0': (sample(_lib.SampleOpts(1, _lib.SAMPLE_TOPP, temperature=0.0, top=0.5)), 'temperature must be positive'),
        'beam_size 17': (beam(_lib.BeamOpts(17, 1)), 'beam_size must be in 1..16'),
        'sample_n neither 1 nor beam_size': (beam(_lib.BeamOpts(3, 2)), 'sample_n must be 1 or beam_size'),
        'teacher steps past ld_tok': (sample(_lib.SampleOpts(1, _lib.SAMPLE_TEACHER, steps=T + 1), ld_tok=T, tokens=tok), 'steps out of range'),
    }
    for name, (make, expected) in cases.items():
        msgs = {f: refused(m, make(m)) for f, m in ms.items()}
        assert expected in msgs['updown'], (name, msgs)
        assert len(set(msgs.values())) == 1, (name, msgs)

    groups = {'updown': 2, 'att2in2': 2, 'newfc': 2, 'aoa': 10, 'transformer': 2}
    msgs = {}
    for f, n in groups.items():
        m = ms[f]
        table = (ctypes.c_void_p * (n + 1))()
        msgs[f] = refused(m, lambda lib: getattr(lib, 'capb200_%s_set_grad_events' % m._abi)(m._engine, table, n + 1))
        assert msgs[f] == 'the engine has %d gradient groups' % n
    assert len({re.sub(r'\d+', 'N', s) for s in msgs.values()}) == 1
