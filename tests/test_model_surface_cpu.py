"""CPU: what the Python surface of the five engine families and the ensemble hands the C ABI, through a recording stand-in for
libcapb200.

Every C call a model makes (engine life cycle, weight binding, the fused XE / SCST steps, the autograd entry points, decoding and the
gradient-event registration) is recorded with its entry name, its scalars and every field of every struct it passes, nested structs and
arrays included.  Each pointer is replaced by what it points into: a parameter or buffer name, ``grad:<slot>`` (the persistent flat
gradient buffer of the fused steps), ``in:<input>``, an engine handle, or ``buf<k>`` for a buffer the call allocates (numbered by first
appearance within the call).  The public methods' signatures and the keys and shapes of the step results are recorded too.  The
transcript must equal tests/golden/model_surface_transcript.json, where every large struct stands as a digest of its content (a failing row
is printed in full); regenerate it with ``python tests/test_model_surface_cpu.py --write``.

Each case seeds torch first and leaves seed=None in some calls, so the order of the host-side seed draws is pinned as well.
"""
import contextlib
import ctypes
import gc
import hashlib
import inspect
import json
import os
import sys
from unittest import mock

import numpy as np
import pytest
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)

import imagecaptioning.pytorch_b200 as b200                     # noqa: E402
from imagecaptioning.pytorch_b200 import _lib, models          # noqa: E402
from imagecaptioning.pytorch_b200 import synthetic as syn      # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'model_surface_transcript.json')
CFG = dict(V=20, E=16, H=16, A=8, F_fc=12, F_att=12, T=6)
SIZES = {'transformer': dict(CFG, E=16, H=32, A=2)}            # d_model, d_ff, layers per stack
B, R, SPI = 2, 3, 2
FAMILIES = ['updown', 'att2in2', 'newfc', 'aoa', 'transformer']
STREAM, CIDER_TABLE, HANDLE_BASE = 0x5EED0000, 0xC1DE0000, 0x7E570000


class _Ptr(int):
    """An address still to be named."""


class _Recorder:
    """Stands in for the loaded library: every capb200_* symbol records its call and succeeds; *_create returns a fresh handle."""

    def __init__(self):
        self.calls = None                # None: not recording
        self.handles = {}

    def __getattr__(self, name):
        if not name.startswith('capb200_'):
            raise AttributeError(name)
        argtypes = _lib.SIGNATURES[name][1]

        def call(*args):
            if name == 'capb200_last_error':
                return b''
            ret = 0
            if name.endswith('_create'):
                ret = HANDLE_BASE + 0x100 * (len(self.handles) + 1)
                self.handles[ret] = 'handle:%s#%d' % (name[len('capb200_'):-len('_create')], len(self.handles))
            if self.calls is not None:
                assert len(args) == len(argtypes), name
                self.calls.append([name[len('capb200_'):], [_ser(a, t) for a, t in zip(args, argtypes)]])
            return ret
        return call


def _is_ptr_type(t):
    return t is ctypes.c_void_p or (isinstance(t, type) and issubclass(t, ctypes._Pointer))


def _ser(v, ctype=None):
    """A ctypes argument or field as JSON-able data, with addresses left as _Ptr.  Null and zero fields of structs are left out."""
    if v is None:
        return None
    if type(v).__name__ == 'CArgObject':             # ctypes.byref(struct)
        return _ser(v._obj)
    if isinstance(v, ctypes._Pointer):
        return _ser(v.contents) if v else None
    if isinstance(v, ctypes.Structure):
        out = {}
        for f, t in type(v)._fields_:
            s = _ser(getattr(v, f), t)
            if s is not None and not (type(s) in (int, float) and s == 0):
                out[f] = s
        return out
    if isinstance(v, ctypes.Array):
        return [_ser(e, v._type_) for e in v]
    if isinstance(v, bool):
        return int(v)
    if isinstance(v, int):
        return _Ptr(v) if _is_ptr_type(ctype) else v
    if isinstance(v, float):
        return v
    raise TypeError('unexpected ctypes value %r' % (v,))


def _resolve(x, known, local, path=None):
    """Names the addresses; a struct field pointing at the flat gradient of its own slot (path) reads 'grad'."""
    if isinstance(x, _Ptr):
        p = int(x)
        name = known[p] if p in known else local.setdefault(p, 'buf%d' % len(local))
        return 'grad' if path and name == 'grad:' + '/'.join(map(str, path)) else name
    if isinstance(x, dict):
        return {k: _resolve(v, known, local, (path or ()) + (k,)) for k, v in x.items()}
    if isinstance(x, list):
        return [_resolve(v, known, local, None if path is None else path + (i,)) for i, v in enumerate(x)]
    return x


def _leaves(x, path=()):
    if isinstance(x, dict):
        for k, v in x.items():
            yield from _leaves(v, path + (k,))
    elif isinstance(x, list):
        for i, v in enumerate(x):
            yield from _leaves(v, path + (i,))
    else:
        yield path, x


REC = _Recorder()


def _enter_device(self, device):
    models._tls.dev = 0
    if self._store.owner is None:
        self._store.owner = id(self)
    return _lib.load()


@contextlib.contextmanager
def _stand_in():
    with mock.patch.object(_lib, 'load', lambda: REC), mock.patch.object(_lib, 'current_stream', lambda: STREAM), \
            mock.patch.object(models.B200CaptionModel, '_enter_device', _enter_device), \
            mock.patch.object(torch.cuda, 'device', lambda d: contextlib.nullcontext()):
        yield


class _Table:
    """The CIDEr-D table argument of scst_step."""

    def handle_for(self, refs):
        return CIDER_TABLE


def _model(family):
    cfg = SIZES.get(family, CFG)
    opt = syn.model_opt(family, heads=2, **cfg)
    opt.vocab = dict(opt.vocab, **{'3': 'the', '5': 'a'})          # bad endings for remove_bad_endings
    torch.manual_seed(0)
    return b200.setup(opt, numeric_mode='tc_f16x3')


class _Inputs:
    def __init__(self):
        g = torch.Generator().manual_seed(3)
        T, V = CFG['T'], CFG['V']
        self.fc = torch.randn(B, CFG['F_fc'], generator=g)
        self.att = torch.randn(B, R, CFG['F_att'], generator=g)
        self.att_masks = torch.tensor([[1.0, 1.0, 0.0], [1.0, 0.0, 0.0]])
        self.labels = torch.zeros(B, SPI, T + 2, dtype=torch.long)
        self.masks = torch.zeros(B, SPI, T + 2)
        for r, n in enumerate((3, 5, 2, 4)):
            self.labels.view(-1, T + 2)[r, 1:1 + n] = torch.randint(1, V + 1, (n,), generator=g)
            self.masks.view(-1, T + 2)[r, :n + 2] = 1.0
        self.gts = [np.random.RandomState(i).randint(1, V + 1, size=(3, 7)).astype(np.int64) for i in range(B)]
        self.forced = torch.randint(1, V + 1, (B * SPI, T), generator=g)
        self.forced_baseline = torch.randint(1, V + 1, (B, T), generator=g)

    def tensors(self):
        return {k: v for k, v in vars(self).items() if isinstance(v, torch.Tensor)}


def _known(model, x):
    known = {STREAM: 'stream', CIDER_TABLE: 'cider_table', **REC.handles}
    for n, t in x.tensors().items():
        known.setdefault(t.data_ptr(), 'in:' + n)
    for m in list(getattr(model, 'models', [])) + [model]:       # an ensemble member's weights by the member's own names
        for n, t in list(m.named_parameters()) + list(m.named_buffers()):
            known.setdefault(t.data_ptr(), n)
    for m in [model] + list(getattr(model, 'models', [])):
        for slot in m._store.slots.values():
            if slot['flat'] is not None:
                for n, t in slot['flat'].by_name.items():
                    known.setdefault(t.data_ptr(), 'grad:' + n)
    return known


def _summary(v, known):
    """Result of a surface call: tensors by shape and dtype, gradient maps by parameter name and slot."""
    if isinstance(v, torch.Tensor):
        return ['tensor', list(v.shape), str(v.dtype)]
    if isinstance(v, dict):
        out = {}
        for k, w in v.items():
            if isinstance(k, torch.Tensor):
                out[known[k.data_ptr()]] = known.get(w.data_ptr(), 'unnamed')
            else:
                out[k] = _summary(w, known)
        return out
    if isinstance(v, (list, tuple)):
        return [_summary(w, known) for w in v]
    if v is None or isinstance(v, (int, float, str)):
        return v
    return type(v).__name__


# ---- cases: each takes (model, inputs, log) and logs the results of its surface calls ------------------------------------------------

def _engine(m, x, log):
    with torch.no_grad():
        log(m(x.fc, x.att, None, opt={'sample_method': 'greedy'}, mode='sample'))       # create, bind, decode
        log(m(x.fc, x.att, None, opt={'sample_method': 'greedy'}, mode='sample'))       # bound: no re-bind
        next(iter(m.parameters())).add_(0.0)                                           # a new version: re-bind
        log(m(x.fc, x.att, None, opt={'sample_method': 'greedy'}, mode='sample'))
    log(m.launch_count)
    m.__del__()


def _xe(m, x, log):
    m.train()
    log(m.xe_step(x.fc, x.att, x.labels, x.masks, label_smoothing=0.2))
    m.ss_prob = 0.25
    log(m.xe_step(x.fc, x.att, x.labels, x.masks, drop_prob=0.3, seed=11, upstream=0.5, att_masks=x.att_masks, keep_rows=3))


def _scst(m, x, log):
    m.train()
    t = _Table()
    log(m.scst_step(x.fc, x.att, x.gts, t, 2))
    log(m.scst_step(x.fc, x.att, x.gts, t, 3, temperature=0.7, seed=5, baseline='leave_one_out', sample_method='top3', reward_weights=(1.0, 0.5),
                    keep_rows=4, att_masks=x.att_masks))
    log(m.scst_step(x.fc, x.att, x.gts, t, 2, drop_prob=0.2, upstream=2.0, forced_tokens=x.forced, forced_baseline=x.forced_baseline))


def _errors(m, x, log):
    m.train()
    t = _Table()
    for call in (lambda: m.scst_step(x.fc, x.att, x.gts, t, 2, baseline='bogus'),
                 lambda: m.scst_step(x.fc, x.att, x.gts, t, 2, baseline='leave_one_out', baseline_method='sample'),
                 lambda: m.scst_step(x.fc, x.att, x.gts, t, 2, sample_method='top999'),
                 lambda: m.scst_step(x.fc, x.att, [x.gts[0], np.zeros((0, 7), np.int64)], t, 2, reward_weights=(1.0, 1.0)),
                 lambda: m.xe_step(x.fc, x.att, x.labels.view(B * SPI, -1)[:3], x.masks.view(B * SPI, -1)[:3]),
                 lambda: m(x.fc, x.att, None, opt={'beam_size': 4, 'group_size': 2, 'sample_n': 2}, mode='sample')):
        try:
            log(call())
        except (ValueError, NotImplementedError, AssertionError) as e:
            log('raises ' + type(e).__name__)


def _autograd(m, x, log):
    m.autograd = True
    m.train()
    m.ss_prob = 0.25
    lp = m(x.fc, x.att, x.labels[..., :-1], x.att_masks)
    lp.sum().backward()
    log(lp)
    seq, lp = m(x.fc, x.att, None, opt={'sample_method': 'sample', 'sample_n': 2}, mode='sample')
    lp.sum().backward()
    log((seq, lp))


def _decode(m, x, log, diverse=True):
    m.eval()
    with torch.no_grad():
        log(m(x.fc, x.att, x.att_masks, opt={'sample_method': 'top5', 'sample_n': 2, 'temperature': 0.8, 'block_trigrams': 1, 'remove_bad_endings': 1},
              mode='sample'))
        log(m._sample(x.fc, x.att, None, opt={'sample_n': 2}, forced_tokens=x.forced))
        log(m(x.fc, x.att, x.labels, x.att_masks))
        log(m(x.fc, x.att, x.att_masks, opt={'beam_size': 3, 'sample_n': 3, 'length_penalty': 'wu_0.5', 'remove_bad_endings': 1,
                                             'decoding_constraint': 1}, mode='sample'))
        m.done_beams[1][2]['logps']          # the record call (the lengths are the stand-in's garbage)
        if diverse:
            log(m(x.fc, x.att, None, opt={'beam_size': 4, 'group_size': 2, 'sample_n': 2, 'diversity_lambda': 0.3, 'temperature': 0.9},
                  mode='sample'))
            m.done_beams[0][3]['logps']          # the record call (the lengths are the stand-in's garbage)


def _grad_sync(m, x, log):
    m.train()
    m._grad_sync_on = True
    log(m.xe_step(x.fc, x.att, x.labels, x.masks))
    m._grad_sync_on = False
    log(m.xe_step(x.fc, x.att, x.labels, x.masks))


CASES = {'engine': _engine, 'xe': _xe, 'scst': _scst, 'errors': _errors, 'autograd': _autograd, 'decode': _decode, 'grad_sync': _grad_sync}


def _ensemble_decode(m, x, log):
    with torch.no_grad():
        log(m(x.fc, x.att, x.att_masks, opt={'sample_method': 'greedy'}, mode='sample'))
        log(m(x.fc, x.att, None, opt={'sample_method': 'sample', 'sample_n': 2}, mode='sample'))
        log(m(x.fc, x.att, x.att_masks, opt={'beam_size': 3, 'sample_n': 1}, mode='sample'))
        m.done_beams[1][0]['logps']          # the record call (the lengths are the stand-in's garbage)
        log(m(x.fc, x.att, x.labels))
    log(m.launch_count)
    m.__del__()


def _ensemble():
    return b200.B200AttEnsemble([_model(f) for f in ('updown', 'att2in2', 'newfc', 'aoa')], weights=[1.0, 2.0, 0.5, 1.0])


def _run(case):
    """The transcript of one case: [[entry, args] ...] with a ['result', ...] row after each surface call."""
    family, kind = case.split('/')
    with _stand_in():
        gc.collect()                    # models of earlier cases destroy their engines now, not inside this record
        REC.handles = {}
        model = _ensemble() if family == 'ensemble' else _model(family)
        x = _Inputs()
        rows = []
        REC.calls = []

        def log(res):
            rows.append((len(REC.calls), res))
        fn = _ensemble_decode if family == 'ensemble' else CASES[kind]
        torch.manual_seed(1234)
        if kind == 'decode' and family in ('newfc', 'transformer'):
            fn(model, x, log, diverse=False)
        else:
            fn(model, x, log)
        calls, REC.calls = REC.calls, None
        known = _known(model, x)
        out, at = [], 0
        for n, res in rows:
            for name, args in calls[at:n]:
                out.append([name, _resolve(args, known, {})])
            out.append(['result', _summary(res, known)])
            at = n
        out += [[name, _resolve(args, known, {})] for name, args in calls[at:]]
        # a step's {parameter: gradient} reads as one line when each parameter's gradient is the flat slot of the field it is bound to
        bound = next(({p: '/'.join(map(str, path)) for path, p in _leaves(args[1])} for name, args in out if name.endswith('_bind_weights')), {})
        for row in out:
            g = row[1].get('grads') if row[0] == 'result' and isinstance(row[1], dict) else None
            if g and all(v == 'grad:' + bound.get(k, '?') for k, v in g.items()):
                row[1]['grads'] = 'the slot of each of %d bound parameters' % len(g)
        for m in [model] + list(getattr(model, 'models', [])):
            m.__del__()                 # the stand-in's handles must never reach the real library
        del model, x, rows
        gc.collect()
    return out


def _signatures():
    out = {}
    for cls in (b200.B200UpDownModel, b200.B200Att2in2Model, b200.B200NewFCModel, b200.B200AoAModel, b200.B200TransformerModel, b200.B200AttEnsemble):
        for meth in ('xe_step', 'scst_step', '_call_sample', '_call_beam', '_call_beam_diverse', '_call_record'):
            if hasattr(cls, meth):
                out['%s.%s' % (cls.__name__, meth)] = str(inspect.signature(getattr(cls, meth)))
    return out


CASE_IDS = ['%s/%s' % (f, k) for f in FAMILIES for k in CASES] + ['ensemble/decode']


def _digest(x):
    """Replaces every struct or map whose JSON is longer than 100 characters (innermost first) by '#' and 16 hex digits of its SHA-256: the
    weights and gradient structs (hundreds of fields at a few layers) are compared exactly without being spelled out in the golden file."""
    if isinstance(x, list):
        return [_digest(v) for v in x]
    if not isinstance(x, dict):
        return x
    x = {k: _digest(v) for k, v in x.items()}
    key = json.dumps(x)
    return x if len(key) <= 100 else '#' + hashlib.sha256(key.encode()).hexdigest()[:16]


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)


def test_signatures():
    assert _signatures() == _golden()['signatures']


@pytest.mark.parametrize('case', CASE_IDS)
def test_transcript(case):
    want = _golden()['cases'][case]
    got = json.loads(json.dumps(_run(case)))
    for i, (a, b) in enumerate(zip(got, want)):
        assert _digest(a) == b, 'row %d of %s differs:\n got  %s\n want %s' % (i, case, json.dumps(a), json.dumps(b))
    assert len(got) == len(want)


if __name__ == '__main__':
    if '--write' not in sys.argv:
        sys.exit('usage: python tests/test_model_surface_cpu.py --write   (rewrites %s)' % os.path.relpath(GOLDEN, REPO))
    cases = {c: _digest(json.loads(json.dumps(_run(c)))) for c in CASE_IDS}
    with open(GOLDEN, 'w') as f:            # one call per line, so that a change reads as a line diff
        f.write('{"signatures": %s,\n "cases": {\n' % json.dumps(_signatures(), indent=1))
        f.write(',\n'.join('  %s: [\n%s]' % (json.dumps(c), ',\n'.join('   ' + json.dumps(row) for row in rows)) for c, rows in cases.items()))
        f.write('}}\n')
    print('wrote %s (%d cases)' % (GOLDEN, len(CASE_IDS)))
