"""Host-side mirror of the reference's model surface for the decode hot path.

``B200UpDownModel`` / ``B200NewFCModel`` present exactly what ``captioning.models.setup(opt)`` returns for
``caption_model in ('updown', 'topdown', 'newfc')`` (captioning/models/__init__.py:20-73):

  * the same constructor argument (``opt`` namespace) and attributes (vocab_size, seq_length, bos/eos/pad/unk_idx,
    vocab, bad_endings_ix, ss_prob, done_beams)                                   AttModel.py:52-97
  * the same ``state_dict`` keys and tensor layouts, so reference checkpoints load unchanged (tools/train.py:79-80)
  * ``forward(*args, mode=...)`` dispatching to ``_forward`` / ``_sample`` (/ ``_sample_beam``)   CaptionModel.py:29-33
  * ``_sample(fc_feats, att_feats, att_masks=None, opt={})`` -> (seq int64 [B*n, T], seqLogprobs fp32 [B*n, T, V+1])
    and ``self.done_beams`` after beam search                                      AttModel.py:218-352

The parameters are ordinary ``nn.Parameter``s owned by PyTorch; every timestep of every decode runs in the hand-written
sm_90a kernels behind the C ABI (include/capb200.h).  Nothing here computes on the CPU and nothing falls back to
PyTorch ops: unsupported decode options raise.
"""
from __future__ import annotations

import ctypes
import threading
from collections.abc import Mapping
from typing import Optional

import torch
import torch.nn as nn

from . import _lib

BAD_ENDINGS = ['a', 'an', 'the', 'in', 'for', 'at', 'of', 'with', 'before', 'after', 'on', 'upon', 'near', 'to', 'is', 'are', 'am', 'the']

_PENALTY = {'': 0, 'wu': 1, 'avg': 2}


class _DoneBeam(Mapping):
    """One finished hypothesis, dict-compatible with CaptionModel.py:190-195.  ``logps`` ([len, V+1]) is gathered from the
    engine's per-step slab on first access instead of being copied for every beam of every image."""

    def __init__(self, owner, image, rank, seq, p, raw):
        self._owner, self._image, self._rank = owner, image, rank
        self._seq, self._p, self._raw = seq, p, raw
        self._logps = None

    def _materialise(self):
        if self._logps is None:
            self._logps = self._owner._beam_logps(self._image, self._rank)[: self._seq.shape[0]]
        return self._logps

    def __getitem__(self, key):
        if key == 'seq':
            return self._seq
        if key == 'p':
            return self._p
        if key == 'logps':
            return self._materialise()
        if key == 'unaug_p':
            return float(self._materialise().sum().item())
        if key == 'sum_logp':          # extension: the raw (un-penalised) running sum
            return self._raw
        raise KeyError(key)

    def __iter__(self):
        return iter(('seq', 'logps', 'unaug_p', 'p'))

    def __len__(self):
        return 4


class _EngineStore:
    """Per-device engine handles of one model, shared BY REFERENCE between the module and the shallow replicas nn.DataParallel makes on
    every forward (replicate() copies __dict__), so each GPU keeps its engine, workspaces and CUDA graphs across steps.  Only the
    module that created the store frees the engines."""

    def __init__(self, owner):
        self.owner = id(owner)
        self.lock = threading.RLock()
        self.slots = {}

    def slot(self, dev):
        with self.lock:
            return self.slots.setdefault(dev, {'engine': None, 'key': None, 'versions': None, 'keepalive': None, 'flat': None, 'bufs': {}})

    def __deepcopy__(self, memo):
        fresh = _EngineStore(None)
        fresh.owner = None          # claimed by the copy at its first _ensure_engine
        return fresh

    def __getstate__(self):
        return {}

    def __setstate__(self, state):
        self.owner, self.lock, self.slots = None, threading.RLock(), {}


_tls = threading.local()           # device index the calling thread is decoding on (set by _ensure_engine)


def _on_device(fn):
    """Runs a call surface with the tensors' device current: the C ABI launches on the current device's stream and never calls
    cudaSetDevice itself, so a model living on cuda:1 while cuda:0 is current (model.to('cuda:1') without set_device) would otherwise launch
    on the wrong device with foreign pointers.  PyTorch modules handle that case transparently; so does this."""
    import functools

    @functools.wraps(fn)
    def wrapped(self, *args, **kwargs):
        dev = next((a.device for a in args if isinstance(a, torch.Tensor) and a.is_cuda), None)
        if dev is None:
            return fn(self, *args, **kwargs)
        with torch.cuda.device(dev):
            return fn(self, *args, **kwargs)
    return wrapped


def sampling_method(sample_method):
    """The engine's form of a reference ``sample_method`` (CaptionModel.sample_next_word, CaptionModel.py:370-407): (CAPB200_SAMPLE_* code,
    top, gumbel).  'gumbel' is the argmax of logprobs + Gumbel noise, a multinomial draw at temperature 1 (the caller pins the temperature);
    'top<x>' is nucleus sampling for 0 < x < 1 and top-k sampling with k = int(x) otherwise."""
    if sample_method == 'greedy':
        return _lib.SAMPLE_GREEDY, 0.0, False
    if sample_method == 'sample':
        return _lib.SAMPLE_MULTINOMIAL, 0.0, False
    if sample_method == 'gumbel':
        return _lib.SAMPLE_MULTINOMIAL, 0.0, True
    if isinstance(sample_method, str) and sample_method.startswith('top'):
        top = float(sample_method[3:])
        if not top > 0:
            raise ValueError('sample_method %r: top-k needs k >= 1, nucleus sampling 0 < p < 1' % sample_method)
        return (_lib.SAMPLE_TOPP if top < 1 else _lib.SAMPLE_TOPK), top, False
    raise NotImplementedError("sample_method %r is out of scope of the engine" % sample_method)


def _scst_sampler(sample_method, baseline_method, forced_baseline, loo, B, T, V1, temperature, dev):
    """(capb200_sampler_opts pointer or None, what must outlive the call, the samples' temperature) of a fused SCST step.  The default
    multinomial samples with the greedy baseline pass no struct, so the step runs exactly as it did before samplers were selectable."""
    if sample_method == 'sample' and baseline_method == 'greedy' and forced_baseline is None:
        return None, None, temperature
    train, train_top, gumbel = sampling_method(sample_method)
    base, base_top, _ = sampling_method(baseline_method)
    for top in (train_top, base_top):
        if top >= 1 and int(top) > V1:
            raise ValueError('top-k sampling needs k <= vocab_size + 1 (%d), got %d' % (V1, int(top)))
    if loo and (base != _lib.SAMPLE_GREEDY or forced_baseline is not None):
        raise ValueError("the leave-one-out baseline draws no baseline captions: baseline_method belongs to baseline='greedy'")
    fb = None
    if forced_baseline is not None:       # replay given baseline captions (parity tests against the reference's own draw)
        fb = forced_baseline.detach().to(device=dev, dtype=torch.long).contiguous()
        assert fb.shape == (B, T)
    so = _lib.SamplerOpts(train, train_top, base, base_top, _lib.ptr(fb))
    return ctypes.pointer(so), (so, fb), 1.0 if gumbel else temperature


def _slot_property(field):
    def get(self):
        return self._store.slot(getattr(_tls, 'dev', None))[field]

    def put(self, value):
        self._store.slot(getattr(_tls, 'dev', None))[field] = value
    return property(get, put)


def _slot_name(path):
    return '/'.join(str(x) for x in path)


class B200CaptionModel(nn.Module):
    """Common machinery: engine life-cycle, weight binding, the call surfaces and the fused training steps.  The per-family data below
    defaults to the UpDown engine's (UpDown, Att2in2, NewFC); AoANet and the Transformer have engines of their own."""

    family = None           # _lib.FAMILY_*
    family_name = ''
    _abi = 'engine'         # capb200_<abi>_create / _destroy / _bind_weights / _launch_count / _set_grad_events
    _takes_fc = True        # the engine's entry points take the fc features ahead of the region features
    _entry = None           # capb200_<entry>_{xe,scst}_{step,vjp}: the training entry points (None: the model does not train)
    _weights_struct, _grads_struct = _lib.Weights, None
    _bind_only = frozenset()                # slot paths that are bound as weights but have no gradient
    _parallel_pass = False  # the teacher-forced pass computes every position in one pass: no scheduled sampling, no early stop

    def __init__(self, opt, numeric_mode: Optional[str] = None):
        super().__init__()
        self.vocab_size = opt.vocab_size
        self.input_encoding_size = opt.input_encoding_size
        self.rnn_size = opt.rnn_size
        self.num_layers = getattr(opt, 'num_layers', 1)
        self.drop_prob_lm = getattr(opt, 'drop_prob_lm', 0.5)
        self.seq_length = getattr(opt, 'max_length', 20) or opt.seq_length
        self.fc_feat_size = opt.fc_feat_size
        self.att_feat_size = opt.att_feat_size
        self.att_hid_size = opt.att_hid_size
        self.bos_idx = getattr(opt, 'bos_idx', 0)
        self.eos_idx = getattr(opt, 'eos_idx', 0)
        self.pad_idx = getattr(opt, 'pad_idx', 0)
        self.unk_idx = getattr(opt, 'unk_idx', None)
        if (self.bos_idx, self.eos_idx, self.pad_idx) != (0, 0, 0):
            raise NotImplementedError('capb200 engine assumes bos = eos = pad = 0 (AttModel.py:65-67 defaults)')
        if getattr(opt, 'use_bn', 0):
            raise NotImplementedError('use_bn is not on the engine decode path')
        # AttModel.py:87-92; k <= 0 makes the reference's reduce fail on an empty list
        self.logit_layers = int(getattr(opt, 'logit_layers', 1))
        if self.logit_layers < 1:
            raise ValueError('logit_layers must be >= 1 (got %d)' % self.logit_layers)
        self.ss_prob = 0.0
        self.vocab = opt.vocab
        self.bad_endings_ix = [int(k) for k, v in self.vocab.items() if v in BAD_ENDINGS]
        self.numeric_mode = numeric_mode or getattr(opt, 'b200_numeric_mode', 'tc_f16x3')
        if self.numeric_mode not in _lib.MODES:
            raise ValueError('numeric_mode must be one of %s' % sorted(_lib.MODES))
        self.done_beams = []
        self._store = _EngineStore(self)
        # differentiable _forward / _sample (the autograd entry points, include/capb200.h: capb200_vjp_opts); off = the calls as before
        self.autograd = bool(getattr(opt, 'b200_autograd', 0))

    # ---- the output head (AttModel.py:87-92) -------------------------------------------------------------------------
    def _make_logit(self):
        """self.logit as AttModel builds it: the vocabulary Linear, or for logit_layers = k > 1 k - 1 [Linear(H, H), ReLU, Dropout(0.5)]
        blocks ahead of it (state_dict keys logit.0, logit.3, ..., logit.{3(k-1)}).  The engine runs the hidden layers outside the recurrence,
        in every decode and every training call (their gradients are group 0, with the vocabulary Linear's)."""
        H, V1 = self.rnn_size, self.vocab_size + 1
        if self.logit_layers == 1:
            return nn.Linear(H, V1)
        hidden = [m for _ in range(self.logit_layers - 1) for m in (nn.Linear(H, H), nn.ReLU(), nn.Dropout(0.5))]
        return nn.Sequential(*hidden, nn.Linear(H, V1))

    @property
    def _vocab_logit(self):
        """The vocabulary Linear of self.logit (its last layer)."""
        return self.logit if isinstance(self.logit, nn.Linear) else self.logit[-1]

    def _head_named(self):
        """[(state_dict name, tensor)] of the logit head's hidden layers, weight then bias per layer; empty for logit_layers = 1 and for the
        Transformer (which has no self.logit)."""
        head = getattr(self, 'logit', None)
        if not isinstance(head, nn.Sequential):
            return []
        return [('logit.%d.%s' % (3 * i, f), getattr(head[3 * i], f)) for i in range(len(head) // 3) for f in ('weight', 'bias')]

    def _bind_head_grads(self, lib, grads, train):
        """Registers the gradient buffers of the head's hidden layers (``grads``: [w_0, b_0, w_1, ...] as _head_named) and its dropout rate
        (Dropout(0.5) in train mode, off in eval mode) with the engine for the training calls that follow."""
        if not grads:
            return
        n = len(grads) // 2
        gw = (ctypes.c_void_p * n)(*[t.data_ptr() for t in grads[0::2]])
        gb = (ctypes.c_void_p * n)(*[t.data_ptr() for t in grads[1::2]])
        _lib.check(getattr(lib, 'capb200_%s_bind_logit_head_grads' % self._abi)(self._engine, gw, gb), '%s_bind_logit_head_grads' % self._abi)
        _lib.check(getattr(lib, 'capb200_%s_set_logit_dropout' % self._abi)(self._engine, 0.5 if train else 0.0), '%s_set_logit_dropout' % self._abi)

    # ---- engine plumbing --------------------------------------------------------------------------------------------
    _engine = _slot_property('engine')
    _engine_key = _slot_property('key')
    _bound_versions = _slot_property('versions')
    _keepalive = _slot_property('keepalive')
    _flat = _slot_property('flat')            # grad_sync.FlatGrads of this device (persistent flat gradient buffer of the fused training steps)
    _bufs = _slot_property('bufs')            # persistent per-shape output buffers of the fused training steps

    def _grad_groups(self, named):
        """The [(slot name, parameter)] of _grad_slots split into lists in the order the engine completes the gradients (include/capb200.h:
        *_set_grad_events): the logit layer and the head's hidden layers first."""
        slots = dict(named)
        first = ('logit_w', 'logit_b') + tuple(n for n, _ in self._head_named())
        return [[(k, slots[k]) for k in first], [(k, v) for k, v in named if k not in first]]

    def _flat_grads(self, device, slots):
        """The persistent flat gradient buffer of this device, its {name: view} table and the engine-recorded group events.  Keyed by name:
        nn.DataParallel replicas carry different Parameter objects every forward but the same names and shapes."""
        from .grad_sync import FlatGrads
        groups = self._grad_groups([(_slot_name(path), p) for path, p in slots] + self._head_named())
        sig = tuple((n, tuple(p.shape)) for g in groups for n, p in g)
        fg = self._flat
        if fg is None or fg.sig != sig:
            fg = FlatGrads([[p for _, p in g] for g in groups], device)
            fg.sig = sig
            fg.by_name = {n: fg.view(p) for g in groups for n, p in g}
            self._flat = fg
        return fg

    def _step_buffers(self, key, make):      # (nn.Module owns the name _buffers)
        bufs = self._bufs
        if key not in bufs:
            bufs.clear()            # one live shape at a time: the buffers are large (the [N, T, V+1] log-prob block)
            bufs[key] = make()
        return bufs[key]

    def _enter_device(self, device):
        """Selects the per-device engine slot for this thread; returns the loaded library."""
        if device.type != 'cuda':
            raise RuntimeError('capb200: the decode engine runs on CUDA devices only (no CPU fallback); got %s' % device)
        _tls.dev = device.index if device.index is not None else torch.cuda.current_device()
        if self._store.owner is None:
            self._store.owner = id(self)
        return _lib.load()

    def _slots(self):
        """[(path of the field in the family's weights / gradient struct, parameter)]; UpDown's engine takes flat structs named by
        _weight_table."""
        return [((name,), t) for name, t in self._weight_table().items()]

    def _grad_slots(self):
        return [(path, p) for path, p in self._slots() if path not in self._bind_only]

    @staticmethod
    def _fill_struct(struct, pairs):
        """Points the fields of a weights / gradient struct at tensors: pairs of (slot path, tensor)."""
        for path, t in pairs:
            dst = struct
            for key in path[:-1]:
                dst = getattr(dst, key) if isinstance(key, str) else dst[key]
            setattr(dst, path[-1], t.data_ptr())

    def _grad_table(self, lib, device, slots=None):
        """The family's gradient struct pointing into the persistent flat buffer, the group events registered with the engine."""
        slots = self._grad_slots() if slots is None else slots
        fg = self._flat_grads(device, slots)
        g = self._grads_struct()
        self._fill_struct(g, [(path, fg.by_name[_slot_name(path)]) for path, _ in slots])
        self._bind_head_grads(lib, [fg.by_name[n] for n, _ in self._head_named()], True)      # the fused steps run in train mode
        # the engine records the group events only for a listener (B200LossWrapper.enable_gradient_sync); without one the whole step may run as a CUDA graph
        table, n = fg.event_table() if getattr(self, '_grad_sync_on', False) else (None, 0)
        _lib.check(getattr(lib, 'capb200_%s_set_grad_events' % self._abi)(self._engine, table, n), '%s_set_grad_events' % self._abi)
        return fg, g

    def _bind_key(self, tensors):
        """What the engine's derived weight copies (fp16 planes, fused QKV blocks, gate tables) were built from.  (data_ptr, _version)
        identifies the contents only for tensors this module owns: the parameters of an nn.DataParallel replica are fresh Broadcast outputs
        every forward (version 0, and the caching allocator hands the same addresses back after an optimizer step), so replicas re-bind on
        every call; the bound tensors are also kept alive so a freed-and-reused address can never look unchanged."""
        if getattr(self, '_is_replica', False) or any(not t.is_leaf for t in tensors):
            return None
        return tuple((t.data_ptr(), t._version) for t in tensors)

    def _ensure_engine(self, device):
        lib = self._enter_device(device)
        key = (_tls.dev, self.numeric_mode)
        if self._engine is None or self._engine_key != key:
            self._destroy_engine()
            cfg = self._cfg()
            with torch.cuda.device(device):
                eng = getattr(lib, 'capb200_%s_create' % self._abi)(ctypes.byref(cfg))
            if not eng:
                raise RuntimeError('capb200 %s_create failed: %s' % (self._abi, lib.capb200_last_error().decode()))
            self._engine, self._engine_key, self._bound_versions = eng, key, None
            if self._head_named():
                _lib.check(getattr(lib, 'capb200_%s_set_logit_layers' % self._abi)(eng, self.logit_layers), '%s_set_logit_layers' % self._abi)
        slots = self._slots()
        head = self._head_named()
        versions = self._bind_key([t for _, t in slots] + [t for _, t in head])
        if versions is None or versions != self._bound_versions:
            keep = []
            for name, t in [(_slot_name(path), t) for path, t in slots] + head:
                if t.device != device or t.dtype != torch.float32:
                    raise RuntimeError('capb200: parameter %s must be a float32 tensor on %s' % (name, device))
                keep.append(t.detach().contiguous())
            w = self._weights_struct()
            self._fill_struct(w, [(path, t) for (path, _), t in zip(slots, keep)])
            _lib.check(getattr(lib, 'capb200_%s_bind_weights' % self._abi)(self._engine, ctypes.byref(w), _lib.current_stream()),
                       '%s_bind_weights' % self._abi)
            if head:
                hk = keep[len(slots):]
                ws = (ctypes.c_void_p * (len(hk) // 2))(*[t.data_ptr() for t in hk[0::2]])
                bs = (ctypes.c_void_p * (len(hk) // 2))(*[t.data_ptr() for t in hk[1::2]])
                _lib.check(getattr(lib, 'capb200_%s_bind_logit_head' % self._abi)(self._engine, ws, bs, _lib.current_stream()),
                           '%s_bind_logit_head' % self._abi)
            self._keepalive = keep
            self._bound_versions = versions
        return lib

    def _cfg(self):
        return _lib.ModelCfg(self.family, self.vocab_size, self.input_encoding_size, self.rnn_size, self.att_hid_size, self.fc_feat_size,
                             self.att_feat_size, self.seq_length, _lib.MODES[self.numeric_mode])

    def _free_engine(self, handle):
        getattr(_lib.load(), 'capb200_%s_destroy' % self._abi)(handle)

    def _destroy_engine(self):
        if self._engine is not None:
            self._free_engine(self._engine)
            self._engine = None

    def __del__(self):
        try:
            store = self.__dict__.get('_store')
            if store is None or store.owner != id(self):
                return                                   # DataParallel replica: the engines belong to the original module
            for slot in store.slots.values():
                if slot['engine'] is not None:
                    self._free_engine(slot['engine'])
                    slot['engine'] = None
        except Exception:
            pass

    @property
    def launch_count(self) -> int:
        return 0 if self._engine is None else int(getattr(_lib.load(), 'capb200_%s_launch_count' % self._abi)(self._engine))

    GEMM_IDS = ('fc_embed', 'att_embed', 'ctx2att', 'fc_gate_bias', 'att_lstm', 'h2att', 'lang_lstm', 'logit', 'newfc_core')

    def set_profiling(self, enable: bool):
        _lib.check(_lib.load().capb200_engine_set_profiling(self._engine, int(enable)), 'set_profiling')

    def read_profile(self, reset=True):
        """{gemm name: (milliseconds, algorithmic FLOPs, launches)} accumulated since the last reset (device-side cudaEvents)."""
        import numpy as np
        ms, fl, calls = np.zeros(9), np.zeros(9), np.zeros(9, dtype=np.int64)
        _lib.check(_lib.load().capb200_engine_read_profile(self._engine, int(reset), ms.ctypes.data, fl.ctypes.data, calls.ctypes.data, 9), 'read_profile')
        return {n: (float(ms[i]), float(fl[i]), int(calls[i])) for i, n in enumerate(self.GEMM_IDS)}

    # ---- reference surface ------------------------------------------------------------------------------------------
    def forward(self, *args, **kwargs):
        mode = kwargs.pop('mode', 'forward')
        return getattr(self, '_' + mode)(*args, **kwargs)

    @staticmethod
    def _f32(t):
        return None if t is None else t.detach().to(torch.float32).contiguous()

    def _clip(self, att_feats, att_masks):
        """clip_att (AttModel.py:106-112): cut the region axis to the longest valid length (one host sync, as the reference)."""
        if att_masks is not None:
            max_len = int(att_masks.detach().long().sum(1).max().item())
            att_feats = att_feats[:, :max_len]
            att_masks = att_masks[:, :max_len]
        return self._f32(att_feats), self._f32(att_masks)

    # why a family has no diverse beam search (None: it has one)
    _no_diverse = None

    def _check_opts(self, opt, beam_size=None, sample_n=None):
        """Refuses what the engine does not run, before any device work.  beam_size / sample_n: the values _sample_beam reads (None: the
        call is not a beam search)."""
        group_size = opt.get('group_size', 1)
        if group_size != 1:
            if beam_size is None or beam_size <= 1:
                raise NotImplementedError('diverse sampling (group_size > 1 with beam_size 1, AttModel._diverse_sample) is out of scope of the engine')
            if self._no_diverse is not None:
                raise NotImplementedError('diverse beam search is not implemented for %s: %s' % (self.family_name, self._no_diverse))
            if group_size < 1 or beam_size % group_size != 0:
                raise NotImplementedError('diverse beam search needs group_size dividing beam_size (got %r, %r)' % (beam_size, group_size))
            if sample_n not in (1, beam_size // group_size):
                raise NotImplementedError('diverse beam search returns sample_n = 1 or beam_size // group_size captions per image (AttModel.py:223)')
            if float(opt.get('diversity_lambda', 0.5)) < 0:
                raise NotImplementedError('diverse beam search needs diversity_lambda >= 0 on the engine (its candidate lists rely on the '
                                          'penalty only lowering log-probs)')
        if opt.get('output_logsoftmax', 1) != 1:
            raise NotImplementedError('output_logsoftmax=0 is out of scope of the engine')

    def _decode_edits(self, opt, device, beam, batch_size=0):
        """The reference's per-step log-prob edits as a capb200_decode_edits (CaptionModel.py:118-120,154-162; AttModel.py:265-332)."""
        ed = _lib.DecodeEdits.none()
        keep = None
        ed.decoding_constraint = 1 if opt.get('decoding_constraint', 0) else 0
        if opt.get('remove_bad_endings', 0) and self.bad_endings_ix:
            keep = torch.tensor(sorted(set(self.bad_endings_ix)), dtype=torch.int32, device=device)
            ed.n_bad_endings, ed.bad_endings = keep.numel(), keep.data_ptr()
        if beam:
            # CaptionModel.py:120 reads opt.get('suppress_UNK', 0); the elif branch lowers unk_idx whatever the flag says (:161-162)
            if opt.get('suppress_UNK', 0) and self.vocab.get(str(self.vocab_size)) == 'UNK':
                ed.unk_col = self.vocab_size
            elif self.unk_idx is not None:
                ed.unk_col = int(self.unk_idx)
            if opt.get('block_trigrams', 0):
                pass                                 # beam search ignores it (the option is only read by _sample, AttModel.py:267)
        elif opt.get('block_trigrams', 0):
            ed.block_trigrams, ed.trigram_rows = 1, int(batch_size)
        return ed, keep

    @_on_device
    def _sample(self, fc_feats, att_feats, att_masks=None, opt={}, forced_tokens=None):
        sample_method = opt.get('sample_method', 'greedy')
        beam_size = opt.get('beam_size', 1)
        temperature = float(opt.get('temperature', 1.0))
        sample_n = int(opt.get('sample_n', 1))
        if self._autograd_active():
            return self._sample_autograd(fc_feats, att_feats, att_masks, opt, forced_tokens)
        if beam_size > 1 and sample_method in ('greedy', 'beam_search'):
            return self._sample_beam(fc_feats, att_feats, att_masks, opt)
        self._check_opts(opt)
        top = 0.0
        if forced_tokens is not None:
            method = _lib.SAMPLE_FORCED
        else:
            method, top, gumbel = sampling_method(sample_method)
            if gumbel:
                temperature = 1.0
        lib = self._ensure_engine(fc_feats.device)
        fc = self._f32(fc_feats)
        att, masks = self._clip(att_feats, att_masks)
        B = fc.shape[0]
        R = att.shape[1] if att is not None and att.dim() == 3 else 1
        N, T, V1 = B * sample_n, self.seq_length, self.vocab_size + 1
        # every (row, step) of both outputs is written by the engine (finished rows get pad / zero rows): no memset of the [N, T, V+1] block
        seq = torch.empty(N, T, dtype=torch.long, device=fc.device)
        logprobs = torch.empty(N, T, V1, dtype=torch.float32, device=fc.device)
        draws = method in (_lib.SAMPLE_MULTINOMIAL, _lib.SAMPLE_TOPK, _lib.SAMPLE_TOPP)
        seed = int(torch.randint(0, 2 ** 62, (1,)).item()) if draws else 0   # follows torch.manual_seed
        edits, keep_bad = self._decode_edits(opt, fc.device, beam=False, batch_size=B)
        so = _lib.SampleOpts(sample_n, method, temperature, seed, T, top, edits)
        tok = None
        if forced_tokens is not None:
            tok = forced_tokens.detach().to(torch.long).contiguous()
            assert tok.shape == (N, T)
        _lib.check(self._call_sample(lib, fc, att, masks, B, R, so, tok, T, seq, logprobs), 'decode_sample')
        return seq, logprobs

    # the decode entry points: capb200_decode_* / capb200_beam_record_logprobs of the UpDown engine, capb200_<abi>_* of the others
    def _decode_fn(self, lib, name):
        return getattr(lib, 'capb200_%s%s' % ('' if self._abi == 'engine' else self._abi + '_', name))

    def _feat_ptrs(self, fc, att):
        return (_lib.ptr(fc), _lib.ptr(att)) if self._takes_fc else (_lib.ptr(att),)

    def _call_sample(self, lib, fc, att, masks, B, R, so, tok, ld_tok, seq, logprobs):
        return self._decode_fn(lib, 'decode_sample')(self._engine, *self._feat_ptrs(fc, att), _lib.ptr(masks), B, R, ctypes.byref(so), _lib.ptr(tok),
                                                     ld_tok, _lib.ptr(seq), _lib.ptr(logprobs), None, _lib.current_stream())

    def _call_beam(self, lib, fc, att, masks, B, R, bo, seq, logprobs, d_seq, d_len, d_p, d_raw):
        return self._decode_fn(lib, 'decode_beam')(self._engine, *self._feat_ptrs(fc, att), _lib.ptr(masks), B, R, ctypes.byref(bo), _lib.ptr(seq),
                                                   _lib.ptr(logprobs), _lib.ptr(d_seq), _lib.ptr(d_len), _lib.ptr(d_p), _lib.ptr(d_raw), _lib.current_stream())

    def _call_beam_diverse(self, lib, fc, att, masks, B, R, do, seq, logprobs, d_seq, d_len, d_p, d_raw):
        return self._decode_fn(lib, 'decode_beam_diverse')(self._engine, *self._feat_ptrs(fc, att), _lib.ptr(masks), B, R, ctypes.byref(do), _lib.ptr(seq),
                                                           _lib.ptr(logprobs), _lib.ptr(d_seq), _lib.ptr(d_len), _lib.ptr(d_p), _lib.ptr(d_raw),
                                                           _lib.current_stream())

    def _call_record(self, lib, image, rank, dst):
        return self._decode_fn(lib, 'beam_record_logprobs')(self._engine, image, rank, _lib.ptr(dst), _lib.current_stream())

    def _teacher_steps(self, seq):
        if self._parallel_pass:
            return seq.shape[1]         # one parallel pass in the reference: every position is computed (TransformerModel.py:340-348)
        # the reference stops at the first column i >= 1 whose labels are all pad (AttModel.py:158-159)
        col_empty = (seq[:, 1:].sum(0) == 0).nonzero()
        return int(col_empty[0].item()) + 1 if col_empty.numel() > 0 else seq.shape[1]

    @_on_device
    def _sample_beam(self, fc_feats, att_feats, att_masks=None, opt={}):
        beam_size = opt.get('beam_size', 10)
        sample_n = opt.get('sample_n', 10)
        group_size = opt.get('group_size', 1)
        self._check_opts(opt, beam_size, sample_n)
        if group_size == 1:
            assert sample_n == 1 or sample_n == beam_size, 'when beam search, sample_n == 1 or beam search'
        assert beam_size <= self.vocab_size + 1
        n_kinds = int(bool(opt.get('decoding_constraint', 0))) + int(bool(opt.get('remove_bad_endings', 0)) and bool(self.bad_endings_ix)) + \
            int((bool(opt.get('suppress_UNK', 0)) and self.vocab.get(str(self.vocab_size)) == 'UNK') or self.unk_idx is not None)
        if beam_size + n_kinds > 16:
            raise NotImplementedError('beam_size + number of active decode edits must be <= 16 on the engine')
        cfg = opt.get('length_penalty', '')
        kind, alpha = (cfg.split('_') + ['0'])[:2] if cfg else ('', '0')
        lib = self._ensure_engine(fc_feats.device)
        fc = self._f32(fc_feats)
        att, masks = self._clip(att_feats, att_masks)
        B = fc.shape[0]
        R = att.shape[1] if att is not None and att.dim() == 3 else 1
        T, V1 = self.seq_length, self.vocab_size + 1
        dev = fc.device
        # all six outputs are written in full by the engine (zero rows / pad beyond each caption's length): no 194 MB memset per call
        seq = torch.empty(B * sample_n, T, dtype=torch.long, device=dev)
        logprobs = torch.empty(B * sample_n, T, V1, dtype=torch.float32, device=dev)
        d_seq = torch.empty(B, beam_size, T, dtype=torch.long, device=dev)
        d_len = torch.empty(B, beam_size, dtype=torch.int32, device=dev)
        d_p = torch.empty(B, beam_size, dtype=torch.float32, device=dev)
        d_raw = torch.empty(B, beam_size, dtype=torch.float32, device=dev)
        edits, keep_bad = self._decode_edits(opt, dev, beam=True)
        bo = _lib.BeamOpts(beam_size, sample_n, _PENALTY[kind], float(alpha), float(opt.get('temperature', 1.0)), edits)
        if group_size == 1:
            _lib.check(self._call_beam(lib, fc, att, masks, B, R, bo, seq, logprobs, d_seq, d_len, d_p, d_raw), 'decode_beam')
        else:       # done_beams[i]: each group's bdash best in group order (CaptionModel.py:207-208)
            do = _lib.DiverseOpts(bo, group_size, float(opt.get('diversity_lambda', 0.5)))
            _lib.check(self._call_beam_diverse(lib, fc, att, masks, B, R, do, seq, logprobs, d_seq, d_len, d_p, d_raw), 'decode_beam_diverse')
        self._last_beam = (d_seq, d_len, d_p, d_raw)
        self.done_beams = _LazyDoneBeams(self, B, beam_size)
        return seq, logprobs

    def _beam_logps(self, image, rank):
        dst = torch.zeros(self.seq_length, self.vocab_size + 1, dtype=torch.float32, device=self._last_beam[0].device)
        _lib.check(self._call_record(_lib.load(), image, rank, dst), 'beam_record_logprobs')
        return dst

    @_on_device
    def _forward(self, fc_feats, att_feats, seq, att_masks=None):
        """Teacher forcing (AttModel.py:126-164).  With model.autograd off this is an inference-style call (plain teacher forcing, no
        grad_fn): training runs in the fused XE step (xe_step / B200LossWrapper), scheduled sampling included.  With it on, under grad, the
        log-probs are differentiable (_forward_autograd)."""
        if self._autograd_active():
            return self._forward_autograd(fc_feats, att_feats, seq, att_masks)
        if self.training and self.ss_prob > 0.0 and torch.is_grad_enabled():
            raise NotImplementedError('scheduled sampling runs inside the fused XE step (B200LossWrapper / model.xe_step), not in a bare _forward call')
        lib = self._ensure_engine(fc_feats.device)
        fc = self._f32(fc_feats)
        att, masks = self._clip(att_feats, att_masks)
        B = fc.shape[0]
        if seq.dim() == 3:
            seq = seq.reshape(-1, seq.shape[2])
        seq = seq.detach().to(torch.long).contiguous()
        spi = seq.shape[0] // B
        L = seq.shape[1]
        if L > self.seq_length + 2:
            raise ValueError('label width %d exceeds what the engine was built for' % L)
        steps = self._teacher_steps(seq)
        R = att.shape[1] if att is not None and att.dim() == 3 else 1
        out = torch.zeros(B * spi, L, self.vocab_size + 1, dtype=torch.float32, device=fc.device)
        so = _lib.SampleOpts(spi, _lib.SAMPLE_TEACHER, 1.0, 0, steps)
        _lib.check(self._call_sample(lib, fc, att, masks, B, R, so, seq, L, None, out), 'forward_teacher')
        return out

    # ---- fused training steps (capb200_<entry>_xe_step / capb200_<entry>_scst_step) ---------------------------------------------------------
    # A family supplies _train_feats, _entry, _rates (its dropout rates, in the order of its option structs), _xe_opts and _scst_opts; the
    # public xe_step / scst_step gather the rates and call the shared bodies.  The defaults are UpDown's, also taken by Att2in2 and NewFC.

    def _train_feats(self, fc_feats, att_feats, att_masks):
        """(what the C entry points take ahead of B, R: (fc, att) or (att,), region masks, B, R): clip_att cuts the region axis to the longest
        valid length (AttModel.py:106-112)."""
        fc = self._f32(fc_feats) if self._takes_fc else None
        att, masks = self._clip(att_feats, att_masks)
        return ((fc, att) if self._takes_fc else (att,)), masks, att.shape[0], att.shape[1]

    def _rates(self, train, drop_prob=None):
        """drop_prob_lm"""
        return (float(self.drop_prob_lm if drop_prob is None else drop_prob),) if train else (0.0,)

    def _xe_opts(self, spi, steps, seed, label_smoothing, upstream, rates, masks, ss_prob, tokens_used, keep_rows, row_loss):
        return _lib.XeOpts(spi, steps, seed, *rates, label_smoothing, upstream, _lib.ptr(masks), ss_prob, _lib.ptr(tokens_used), keep_rows, _lib.ptr(row_loss))

    def _scst_opts(self, sample_n, temperature, seed, upstream, baseline, rates, forced, masks, keep_rows, row_loss, sampler, rw):
        return _lib.ScstOpts(sample_n, temperature, seed, *rates, upstream, baseline, _lib.ptr(forced), _lib.ptr(masks), keep_rows, _lib.ptr(row_loss), sampler, rw)

    def _grads_of(self, fg, slots):
        out = {prm: fg.by_name[_slot_name(path)] for path, prm in slots}
        out.update((prm, fg.by_name[n]) for n, prm in self._head_named())
        return out

    # ---- SCST training step: greedy baseline + sampling with dropout + CIDEr-D reward + RewardCriterion + BPTT -----------------
    @_on_device
    def scst_step(self, fc_feats, att_feats, gts, table, sample_n, temperature=1.0, drop_prob=None, seed=None, upstream=1.0, baseline='greedy',
                  forced_tokens=None, att_masks=None, keep_rows=0, reward_weights=None, sample_method='sample', baseline_method='greedy',
                  forced_baseline=None):
        """Runs one self-critical step entirely on the device (capb200_updown_scst_step and its Att2in2 / NewFC counterparts).  Returns a
        dict with 'loss' (0-dim), 'reward' [N, T], 'sample_seq', 'greedy_seq', 'sample_logprobs' and 'grads' {parameter: gradient tensor}.
        ``baseline='greedy'`` is the self-critical step (loss_wrapper.py:56-73); ``'leave_one_out'`` the 'new_self_critical' structure
        loss (losses.py:168-187): no greedy decode, each sample is scored against the mean of the image's other samples, and the
        result carries 'scores' [B, n] (the raw CIDEr-D values the reference reports as out['reward']).  ``reward_weights`` = (cider, bleu)
        scores each caption with cider * CIDEr-D + bleu * BLEU-4 (opts.py:169-172); None is CIDEr-D alone.  ``sample_method`` draws the
        train-mode samples and ``baseline_method`` the eval-mode baseline (LossWrapper's train_sample_method / sc_sample_method: 'sample',
        'greedy', 'gumbel', 'top<k>', 'top<p>'); the loss and the gradients read the full log-softmax rows whatever the sampler keeps.
        ``forced_baseline`` [B, T] replays given baseline captions, as ``forced_tokens`` [N, T] replays samples."""
        return self._scst_step(fc_feats, att_feats, gts, table, sample_n, self._rates(True, drop_prob), temperature, seed, upstream, baseline,
                               forced_tokens, att_masks, keep_rows, reward_weights, sample_method, baseline_method, forced_baseline)

    def _scst_step(self, fc_feats, att_feats, gts, table, sample_n, rates, temperature, seed, upstream, baseline, forced_tokens, att_masks, keep_rows,
                   reward_weights, sample_method, baseline_method, forced_baseline):
        from .rewards import pack_references, weights_struct
        lead = fc_feats if self._takes_fc else att_feats
        rw = weights_struct(reward_weights, gts)          # refuses a missing reference list before any device work
        sampler, _keep, temperature = _scst_sampler(sample_method, baseline_method, forced_baseline, baseline == 'leave_one_out', lead.shape[0],
                                                    self.seq_length, self.vocab_size + 1, temperature, lead.device)
        lib = self._ensure_engine(lead.device)
        feats, masks, B, R = self._train_feats(fc_feats, att_feats, att_masks)
        dev = feats[0].device
        N, T, V1 = B * sample_n, self.seq_length, self.vocab_size + 1
        refs, offsets, L = pack_references(gts, dev)
        slots = self._grad_slots()
        fg, g = self._grad_table(lib, dev, slots)
        if baseline not in ('greedy', 'leave_one_out'):
            raise ValueError("baseline must be 'greedy' or 'leave_one_out'")
        loo = baseline == 'leave_one_out'
        # outputs live in persistent buffers (overwritten by the next step of the same shape): the step writes every row of every one
        sample_seq, greedy_seq, logprobs, reward, loss = self._step_buffers(('scst', B, sample_n), lambda: (
            torch.zeros(N, T, dtype=torch.long, device=dev), torch.zeros(B, T, dtype=torch.long, device=dev),
            torch.zeros(N, T, V1, dtype=torch.float32, device=dev), torch.empty(N, T, dtype=torch.float32, device=dev),
            torch.empty(1, dtype=torch.float32, device=dev)))
        if seed is None:
            seed = int(torch.randint(0, 2 ** 62, (1,)).item())
        forced = None
        if forced_tokens is not None:       # replay a given draw (parity tests against the reference's own samples)
            forced = forced_tokens.detach().to(device=dev, dtype=torch.long).contiguous()
            assert forced.shape == (N, T)
        row_loss = torch.empty(N, dtype=torch.float32, device=dev) if keep_rows else None      # drop_worst: per-row losses (reduction 'none')
        so = self._scst_opts(sample_n, float(temperature), seed, float(upstream), _lib.BASELINE_LEAVE_ONE_OUT if loo else _lib.BASELINE_GREEDY, rates,
                             forced, masks, int(keep_rows), row_loss, sampler, None if rw is None else ctypes.pointer(rw))
        entry = 'capb200_%s_scst_step' % self._entry
        _lib.check(getattr(lib, entry)(self._engine, *map(_lib.ptr, feats), B, R, ctypes.byref(so), table.handle_for(refs), _lib.ptr(refs),
                                       _lib.ptr(offsets), L, ctypes.byref(g), _lib.ptr(sample_seq), None if loo else _lib.ptr(greedy_seq),
                                       _lib.ptr(logprobs), _lib.ptr(reward), _lib.ptr(loss), _lib.current_stream()), entry[len('capb200_'):])
        return {'loss': loss[0], 'reward': reward, 'sample_seq': sample_seq, 'greedy_seq': None if loo else greedy_seq, 'sample_logprobs': logprobs,
                'grads': self._grads_of(fg, slots), 'seed': seed, 'flat': fg, 'row_loss': row_loss}

    # ---- PPO step: train-mode samples + the frozen old policy's teacher-forced pass + reward + clipped-ratio / KL criterion + BPTT -------------
    @_on_device
    def ppo_step(self, old_model, fc_feats, att_feats, gts, table, sample_n, cliprange=0.2, kl_coef=0.02, temperature=1.0, seed=None, upstream=1.0,
                 forced_tokens=None, att_masks=None, keep_rows=0, reward_weights=None, sample_method='sample', **rates):
        """One PPO step on the device (capb200_<family>_ppo_step; PPOLoss, losses.py:267-357): the train-mode samples of scst_step, the
        teacher-forced pass of ``old_model`` -- a frozen model of the same family and configuration -- in eval mode over [0, seq[:, :-1]],
        the reward (CIDEr-D, or ``reward_weights`` = (cider, bleu)) with the leave-one-out advantage, then
        ``pg_loss + kl_coef * kl_loss`` with the policy ratio clipped to [1 - cliprange, 1 + cliprange] and the gradients of the new policy.
        ``rates`` are the family's dropout rates as its scst_step takes them (drop_prob; the Transformer's dropout; AoANet's drop_attn, ...).
        ``keep_rows`` > 0 is drop_worst: the loss is the mean of the keep_rows smallest per-row losses ('row_loss' holds every row's).
        Returns {'loss', 'pg_loss', 'kl_loss', 'clipfrac' (0-dim), 'scores' [B, n] (the rewarded scores, out['reward']), 'sample_seq',
        'sample_logprobs', 'grads', 'flat', 'seed', 'row_loss'}."""
        from .rewards import pack_references, weights_struct
        if self._entry is None:
            raise NotImplementedError('%s has no fused PPO step' % type(self).__name__)
        if (old_model is self or type(old_model) is not type(self) or bytes(old_model._cfg()) != bytes(self._cfg())
                or getattr(old_model, 'logit_layers', 1) != getattr(self, 'logit_layers', 1)):
            raise ValueError('ppo_step needs an old model of its own with the family and configuration of this one')
        if int(sample_n) < 2:
            raise ValueError("PPO's leave-one-out advantage needs sample_n >= 2")
        lead = fc_feats if self._takes_fc else att_feats
        rw = weights_struct(reward_weights, gts)
        sampler, _keep, temperature = _scst_sampler(sample_method, 'greedy', None, True, lead.shape[0], self.seq_length, self.vocab_size + 1,
                                                    temperature, lead.device)
        lib = self._ensure_engine(lead.device)
        old_model._ensure_engine(lead.device)
        feats, masks, B, R = self._train_feats(fc_feats, att_feats, att_masks)
        dev = feats[0].device
        N, T, V1 = B * sample_n, self.seq_length, self.vocab_size + 1
        refs, offsets, L = pack_references(gts, dev)
        slots = self._grad_slots()
        fg, g = self._grad_table(lib, dev, slots)
        sample_seq, logprobs, scores, stats = self._step_buffers(('ppo', B, sample_n), lambda: (
            torch.zeros(N, T, dtype=torch.long, device=dev), torch.zeros(N, T, V1, dtype=torch.float32, device=dev),
            torch.empty(N, dtype=torch.float32, device=dev), torch.empty(4, dtype=torch.float32, device=dev)))
        if seed is None:
            seed = int(torch.randint(0, 2 ** 62, (1,)).item())
        forced = None
        if forced_tokens is not None:
            forced = forced_tokens.detach().to(device=dev, dtype=torch.long).contiguous()
            assert forced.shape == (N, T)
        row_loss = torch.empty(N, dtype=torch.float32, device=dev) if keep_rows else None
        so = self._scst_opts(sample_n, float(temperature), seed, float(upstream), _lib.BASELINE_LEAVE_ONE_OUT, self._rates(True, **rates), forced, masks,
                             int(keep_rows), row_loss, sampler, None if rw is None else ctypes.pointer(rw))
        po = _lib.PpoOpts(float(cliprange), float(kl_coef))
        entry = 'capb200_%s_ppo_step' % self._entry
        _lib.check(getattr(lib, entry)(self._engine, old_model._engine, *map(_lib.ptr, feats), B, R, ctypes.byref(so), ctypes.byref(po),
                                       table.handle_for(refs), _lib.ptr(refs), _lib.ptr(offsets), L, ctypes.byref(g), _lib.ptr(sample_seq),
                                       _lib.ptr(logprobs), _lib.ptr(scores), *(_lib.ptr(stats[i:i + 1]) for i in range(4)), _lib.current_stream()),
                   entry[len('capb200_'):])
        return {'loss': stats[0], 'pg_loss': stats[1], 'kl_loss': stats[2], 'clipfrac': stats[3], 'scores': scores.view(B, sample_n),
                'sample_seq': sample_seq, 'sample_logprobs': logprobs, 'grads': self._grads_of(fg, slots), 'seed': seed, 'flat': fg,
                'row_loss': row_loss}

    @_on_device
    def xe_step(self, fc_feats, att_feats, labels, masks, label_smoothing=0.0, drop_prob=None, seed=None, upstream=1.0, att_masks=None, keep_rows=0):
        """One cross-entropy step on the device (capb200_updown_xe_step and its Att2in2 / NewFC counterparts): teacher-forced forward over ``labels[..., :-1]`` in train mode,
        LanguageModelCriterion / LabelSmoothing against ``labels[..., 1:]``, ``masks[..., 1:]`` (reduction 'mean'), BPTT.
        Returns {'loss', 'logprobs' [N, L-1, V+1], 'grads' {parameter: gradient}, 'seed'}."""
        return self._xe_step(fc_feats, att_feats, labels, masks, self._rates(True, drop_prob), label_smoothing, seed, upstream, att_masks, keep_rows)

    def _xe_step(self, fc_feats, att_feats, labels, masks, rates, label_smoothing, seed, upstream, att_masks, keep_rows):
        lib = self._ensure_engine((fc_feats if self._takes_fc else att_feats).device)
        feats, region_masks, B, R = self._train_feats(fc_feats, att_feats, att_masks)
        dev = feats[0].device
        if labels.dim() == 3:
            labels = labels.reshape(-1, labels.shape[2])
            masks = masks.reshape(-1, masks.shape[2])
        labels = labels.detach().to(torch.long).contiguous()
        masks = masks.detach().to(torch.float32).contiguous()
        N, Lc = labels.shape
        if N % B != 0 or Lc > self.seq_length + 2 or masks.shape != labels.shape:
            raise ValueError('labels/masks must be [B * seq_per_img, <= seq_length + 2]')
        steps = self._teacher_steps(labels[:, :-1])
        V1 = self.vocab_size + 1
        slots = self._grad_slots()
        fg, g = self._grad_table(lib, dev, slots)
        # a pass that stops at the first all-pad column leaves the rows after it as they are: zero them (a parallel pass writes every position)
        logprobs = (torch.empty if self._parallel_pass else torch.zeros)(N, Lc - 1, V1, dtype=torch.float32, device=dev)
        loss = torch.empty(1, dtype=torch.float32, device=dev)
        if seed is None:
            seed = int(torch.randint(0, 2 ** 62, (1,)).item())
        # scheduled sampling (self.ss_prob, set by the trainer: tools/train.py:147-148): the words actually fed are returned as 'tokens_used'
        ss = 0.0 if self._parallel_pass else float(self.ss_prob)
        tokens_used = torch.zeros(N, Lc - 1, dtype=torch.long, device=dev) if ss > 0.0 else None
        row_loss = torch.empty(N, dtype=torch.float32, device=dev) if keep_rows else None
        xo = self._xe_opts(N // B, steps, seed, float(label_smoothing), float(upstream), rates, region_masks, ss, tokens_used, int(keep_rows), row_loss)
        entry = 'capb200_%s_xe_step' % self._entry
        _lib.check(getattr(lib, entry)(self._engine, *map(_lib.ptr, feats), B, R, ctypes.byref(xo), _lib.ptr(labels), _lib.ptr(masks), Lc,
                                       ctypes.byref(g), _lib.ptr(logprobs), _lib.ptr(loss), _lib.current_stream()), entry[len('capb200_'):])
        return {'loss': loss[0], 'logprobs': logprobs, 'grads': self._grads_of(fg, slots), 'seed': seed, 'flat': fg, 'tokens_used': tokens_used,
                'row_loss': row_loss}


    # ---- autograd path (model.autograd): the forward of the fused training steps, and the backward of an outside dL/dlogprobs -----------
    # capb200_<entry>_xe_vjp / _scst_vjp take the fused steps' features, option structs (_xe_opts, _scst_opts) and gradient struct.

    def _autograd_active(self):
        """model.autograd, grad mode on, and some parameter that wants a gradient."""
        return (getattr(self, 'autograd', False) and self._entry is not None and torch.is_grad_enabled()
                and any(p.requires_grad for _, p in self._grad_slots()))

    @staticmethod
    def _refuse_feature_grads(*feats):
        if any(f is not None and f.requires_grad for f in feats):
            raise NotImplementedError('capb200 autograd: gradients with respect to the features are out of scope (detach them)')

    def _vjp_run(self, form, feats, B, R, make_opts, words, logprobs_shape, dev, greedy=False, out_seq=None, train=True):
        """The closure _EngineVjp calls: run(None) is the forward (log-probs), run(G) the backward of G = dL/dlogprobs (one fresh gradient
        tensor per parameter).  make_opts(replay) builds the option struct: replay=False for the forward, True for the backward, which
        feeds the same words (words()) with the same seed.  ``train``: the logit head's dropout is on."""
        slots = self._grad_slots()
        head = [p for _, p in self._head_named()]
        params = [p for _, p in slots] + head
        entry = 'capb200_%s_%s_vjp' % (self._entry, form)

        def run(G):
            lib = self._ensure_engine(dev)
            lp = torch.zeros(logprobs_shape, dtype=torch.float32, device=dev)
            if G is None:
                opts, vo, g, grads = make_opts(False), _lib.VjpOpts(1, None, int(greedy)), None, None
                self._bind_head_grads(lib, [torch.empty_like(p) for p in head], train)     # not written by a forward-only call
            else:
                G = G.detach().to(torch.float32).contiguous()
                grads = [torch.empty_like(p) for p in params]
                g = self._grads_struct()
                self._fill_struct(g, [(path, t) for (path, _), t in zip(slots, grads)])
                self._bind_head_grads(lib, grads[len(slots):], train)
                opts, vo = make_opts(True), _lib.VjpOpts(0, G.data_ptr(), 0)
            tail = (words(G is not None), logprobs_shape[1] + 1) if form == 'xe' else ()
            seq = out_seq if G is None or out_seq is None else torch.empty_like(out_seq)
            outs = (_lib.ptr(lp),) if form == 'xe' else (_lib.ptr(seq), _lib.ptr(lp))
            args = tuple(map(_lib.ptr, feats)) + (B, R, ctypes.byref(opts), ctypes.byref(vo))
            if form == 'xe':
                args += (_lib.ptr(tail[0]), tail[1])
            _lib.check(getattr(lib, entry)(self._engine, *args, None if g is None else ctypes.byref(g), *outs, _lib.current_stream()),
                       entry[len('capb200_'):])
            return lp if G is None else grads
        return run, params

    def _forward_autograd(self, fc_feats, att_feats, seq, att_masks):
        """Differentiable teacher forcing: train mode runs the fused XE step's forward (its dropout masks and, with ss_prob > 0, its
        scheduled sampling), eval mode the same forward without dropout."""
        self._refuse_feature_grads(fc_feats, att_feats)
        if seq.dim() == 3:
            seq = seq.reshape(-1, seq.shape[2])
        seq = seq.detach().to(torch.long).contiguous()
        N, L = seq.shape
        if L > self.seq_length + 1:
            raise ValueError('label width %d exceeds what the engine trains (seq_length + 1 = %d)' % (L, self.seq_length + 1))
        train = self.training
        seed = int(torch.randint(0, 2 ** 62, (1,)).item()) if train else 0      # where xe_step draws it: torch.manual_seed reproduces both
        feats, masks, B, R = self._train_feats(fc_feats, att_feats, att_masks)
        dev = feats[0].device
        seq = seq.to(dev)
        steps = self._teacher_steps(seq)
        ss = float(self.ss_prob) if train and not self._parallel_pass else 0.0
        tokens_used = torch.zeros(N, L, dtype=torch.long, device=dev) if ss > 0 else None
        pad = seq.new_zeros(N, 1)
        labels = torch.cat([seq, pad], 1)       # [N, L + 1]: the entry points take labels with the target column; it is never read

        def words(replay):
            return torch.cat([tokens_used, pad], 1) if replay and tokens_used is not None else labels

        def make_opts(replay):
            return self._xe_opts(N // B, steps, seed, 0.0, 1.0, self._rates(train), masks, 0.0 if replay else ss, None if replay else tokens_used, 0,
                                 None)
        run, params = self._vjp_run('xe', feats, B, R, make_opts, words, (N, L, self.vocab_size + 1), dev, train=train)
        return _EngineVjp.apply(run, *params)

    def _sample_autograd(self, fc_feats, att_feats, att_masks, opt, forced_tokens):
        """Differentiable sampling: greedy or multinomial draws of the fused SCST step's sampler (train mode: with its dropout, the same
        draws as scst_step for the same seed), seq [B*n, T] and log-probs [B*n, T, V+1] with the reference's finished-row zeros."""
        method = opt.get('sample_method', 'greedy')
        if opt.get('beam_size', 1) > 1 and method in ('greedy', 'beam_search'):
            raise NotImplementedError('capb200 autograd: beam search under grad (train_beam_size > 1) is out of scope')
        self._check_opts(opt)
        edits = [k for k in ('decoding_constraint', 'remove_bad_endings', 'suppress_UNK', 'block_trigrams') if opt.get(k, 0)]
        if edits:
            raise NotImplementedError('capb200 autograd: decode edits (%s) are not differentiated' % ', '.join(edits))
        if forced_tokens is None and method not in ('greedy', 'sample'):
            if method != 'gumbel' and not method.startswith('top'):
                raise NotImplementedError('sample_method %r is out of scope of the engine' % method)
            if self.training:
                raise NotImplementedError('capb200 autograd: sample_method %r in train mode is out of scope (greedy and sample are covered)' % method)
        self._refuse_feature_grads(fc_feats, att_feats)
        sample_n, temperature, train = int(opt.get('sample_n', 1)), float(opt.get('temperature', 1.0)), self.training
        forced = None
        if forced_tokens is None and method not in ('greedy', 'sample'):
            with torch.no_grad():                # eval mode: the decode path draws, the autograd forward replays the draw
                forced, _ = self._sample(fc_feats, att_feats, att_masks, opt)
        elif forced_tokens is not None:
            forced = forced_tokens
        draws = forced is None and method == 'sample'
        seed = int(torch.randint(0, 2 ** 62, (1,)).item()) if train or draws else 0     # where scst_step / _sample draw it
        feats, masks, B, R = self._train_feats(fc_feats, att_feats, att_masks)
        dev = feats[0].device
        N, T = B * sample_n, self.seq_length
        if forced is not None:
            forced = forced.detach().to(device=dev, dtype=torch.long).contiguous()
            assert forced.shape == (N, T)
        seq = torch.zeros(N, T, dtype=torch.long, device=dev)

        def make_opts(replay):
            return self._scst_opts(sample_n, temperature, seed, 1.0, _lib.BASELINE_GREEDY, self._rates(train), seq if replay else forced, masks, 0, None,
                                   None, None)
        run, params = self._vjp_run('scst', feats, B, R, make_opts, None, (N, T, self.vocab_size + 1), dev,
                                    greedy=forced is None and method == 'greedy', out_seq=seq, train=train)
        logprobs = _EngineVjp.apply(run, *params)
        return seq, logprobs


class _EngineVjp(torch.autograd.Function):
    """One node per autograd call of an engine model, with the parameters as inputs.  The backward recomputes the forward instead of
    keeping its tape: the engine's training tape is shared by every training call, and whatever runs between the forward and the backward
    (another forward, a fused step, PPO's old-policy pass) may overwrite it."""

    @staticmethod
    def forward(ctx, run, *params):
        ctx.run = run
        ctx.save_for_backward(*params)          # an in-place update of a weight before the backward raises torch's version error
        return run(None)

    @staticmethod
    def backward(ctx, grad):
        _ = ctx.saved_tensors
        return (None,) + tuple(ctx.run(grad))


class _LazyDoneBeams(list):
    """list[B] of list[beam] of finished-beam records; host copies happen on first indexing (one D2H for the whole batch)."""

    def __init__(self, owner, B, beam):
        super().__init__()
        self._owner, self._B, self._beam, self._built = owner, B, beam, False

    def _build(self):
        if self._built:
            return
        d_seq, d_len, d_p, d_raw = self._owner._last_beam
        lens = d_len.cpu().tolist()
        ps = d_p.double().cpu().tolist()
        raws = d_raw.cpu().tolist()
        for i in range(self._B):
            super().append([_DoneBeam(self._owner, i, j, d_seq[i, j, :lens[i][j]], ps[i][j], raws[i][j]) for j in range(self._beam)])
        self._built = True

    def __getitem__(self, i):
        self._build()
        return super().__getitem__(i)

    def __iter__(self):
        self._build()
        return super().__iter__()

    def __len__(self):
        return self._B


class _UpDownCoreParams(nn.Module):
    """Parameter container with the key names of UpDownCore + Attention (AttModel.py:615-622,719-726)."""

    def __init__(self, opt):
        super().__init__()
        self.att_lstm = nn.LSTMCell(opt.input_encoding_size + opt.rnn_size * 2, opt.rnn_size)
        self.lang_lstm = nn.LSTMCell(opt.rnn_size * 2, opt.rnn_size)
        self.attention = nn.Module()
        self.attention.h2att = nn.Linear(opt.rnn_size, opt.att_hid_size)
        self.attention.alpha_net = nn.Linear(opt.att_hid_size, 1)


class B200UpDownModel(B200CaptionModel):
    """Drop-in for captioning.models.AttModel.UpDownModel (AttModel.py:868-872)."""

    family = _lib.FAMILY_UPDOWN
    family_name = 'updown'
    _entry, _grads_struct = 'updown', _lib.UpdownGrads

    def __init__(self, opt, numeric_mode=None):
        super().__init__(opt, numeric_mode)
        self.num_layers = 2
        V1 = self.vocab_size + 1
        self.embed = nn.Sequential(nn.Embedding(V1, self.input_encoding_size), nn.ReLU(), nn.Dropout(self.drop_prob_lm))
        self.fc_embed = nn.Sequential(nn.Linear(self.fc_feat_size, self.rnn_size), nn.ReLU(), nn.Dropout(self.drop_prob_lm))
        self.att_embed = nn.Sequential(nn.Linear(self.att_feat_size, self.rnn_size), nn.ReLU(), nn.Dropout(self.drop_prob_lm))
        self.logit = self._make_logit()
        self.ctx2att = nn.Linear(self.rnn_size, self.att_hid_size)
        self.core = _UpDownCoreParams(opt)

    def _weight_table(self):
        c = self.core
        return {
            'embed': self.embed[0].weight, 'fc_embed_w': self.fc_embed[0].weight, 'fc_embed_b': self.fc_embed[0].bias,
            'att_embed_w': self.att_embed[0].weight, 'att_embed_b': self.att_embed[0].bias,
            'ctx2att_w': self.ctx2att.weight, 'ctx2att_b': self.ctx2att.bias, 'logit_w': self._vocab_logit.weight, 'logit_b': self._vocab_logit.bias,
            'att_lstm_w_ih': c.att_lstm.weight_ih, 'att_lstm_w_hh': c.att_lstm.weight_hh, 'att_lstm_b_ih': c.att_lstm.bias_ih,
            'att_lstm_b_hh': c.att_lstm.bias_hh, 'lang_lstm_w_ih': c.lang_lstm.weight_ih, 'lang_lstm_w_hh': c.lang_lstm.weight_hh,
            'lang_lstm_b_ih': c.lang_lstm.bias_ih, 'lang_lstm_b_hh': c.lang_lstm.bias_hh,
            'h2att_w': c.attention.h2att.weight, 'h2att_b': c.attention.h2att.bias,
            'alpha_w': c.attention.alpha_net.weight, 'alpha_b': c.attention.alpha_net.bias,
        }


class _Att2in2CoreParams(nn.Module):
    """Parameter container with the key names of Att2in2Core + Attention (AttModel.py:754-768,719-726)."""

    def __init__(self, opt):
        super().__init__()
        self.a2c = nn.Linear(opt.rnn_size, 2 * opt.rnn_size)
        self.i2h = nn.Linear(opt.input_encoding_size, 5 * opt.rnn_size)
        self.h2h = nn.Linear(opt.rnn_size, 5 * opt.rnn_size)
        self.attention = nn.Module()
        self.attention.h2att = nn.Linear(opt.rnn_size, opt.att_hid_size)
        self.attention.alpha_net = nn.Linear(opt.att_hid_size, 1)


class B200Att2in2Model(B200UpDownModel):
    """Drop-in for captioning.models.AttModel.Att2in2Model (AttModel.py:854-859): AttModel without fc_embed, one maxout-LSTM core that
    attends with its previous hidden state.  Decoding, diverse beam search and the fused XE / SCST steps take UpDown's surface; the engine
    runs the Att2in2 core (CAPB200_FAMILY_ATT2IN2)."""

    family = _lib.FAMILY_ATT2IN2
    family_name = 'att2in2'
    _entry, _grads_struct = 'att2in2', _lib.Att2in2Grads

    def __init__(self, opt, numeric_mode=None):
        B200CaptionModel.__init__(self, opt, numeric_mode)
        self.num_layers = 1
        V1 = self.vocab_size + 1
        self.embed = nn.Sequential(nn.Embedding(V1, self.input_encoding_size), nn.ReLU(), nn.Dropout(self.drop_prob_lm))
        self.att_embed = nn.Sequential(nn.Linear(self.att_feat_size, self.rnn_size), nn.ReLU(), nn.Dropout(self.drop_prob_lm))
        self.logit = self._make_logit()
        self.ctx2att = nn.Linear(self.rnn_size, self.att_hid_size)
        self.core = _Att2in2CoreParams(opt)

    def _weight_table(self):
        c = self.core
        return {
            'embed': self.embed[0].weight, 'att_embed_w': self.att_embed[0].weight, 'att_embed_b': self.att_embed[0].bias,
            'ctx2att_w': self.ctx2att.weight, 'ctx2att_b': self.ctx2att.bias, 'logit_w': self._vocab_logit.weight, 'logit_b': self._vocab_logit.bias,
            'h2att_w': c.attention.h2att.weight, 'h2att_b': c.attention.h2att.bias,
            'alpha_w': c.attention.alpha_net.weight, 'alpha_b': c.attention.alpha_net.bias,
            'i2h_w': c.i2h.weight, 'i2h_b': c.i2h.bias, 'h2h_w': c.h2h.weight, 'h2h_b': c.h2h.bias, 'a2c_w': c.a2c.weight, 'a2c_b': c.a2c.bias,
        }


class _MaxoutCoreParams(nn.Module):
    """Parameter container with the key names of FCModel.LSTMCore (FCModel.py:13-23)."""

    def __init__(self, opt):
        super().__init__()
        self.i2h = nn.Linear(opt.input_encoding_size, 5 * opt.rnn_size)
        self.h2h = nn.Linear(opt.rnn_size, 5 * opt.rnn_size)


class B200NewFCModel(B200CaptionModel):
    """Drop-in for captioning.models.AttModel.NewFCModel (AttModel.py:904-945).  The fused XE / SCST steps take UpDown's surface; the
    model reads the fc features only, so ``att_feats`` of any shape (the loader's [B, 0, 0] included) and ``att_masks`` are ignored, as
    in the reference (its _prepare_feature has no clip_att)."""

    family = _lib.FAMILY_NEWFC
    family_name = 'newfc'
    _entry, _grads_struct = 'newfc', _lib.NewfcGrads
    _no_diverse = ("the engine chooses NewFC's fresh-state pass (the image-embedding step, AttModel.py:925-936) per core call, not per row, "
                   "so its groups cannot start at different steps")

    def __init__(self, opt, numeric_mode=None):
        super().__init__(opt, numeric_mode)
        V1 = self.vocab_size + 1
        self.embed = nn.Embedding(V1, self.input_encoding_size)
        self.fc_embed = nn.Linear(self.fc_feat_size, self.input_encoding_size)
        self.logit = self._make_logit()
        self._core = _MaxoutCoreParams(opt)

    def _weight_table(self):
        return {
            'embed': self.embed.weight, 'fc_embed_w': self.fc_embed.weight, 'fc_embed_b': self.fc_embed.bias,
            'logit_w': self._vocab_logit.weight, 'logit_b': self._vocab_logit.bias,
            'i2h_w': self._core.i2h.weight, 'i2h_b': self._core.i2h.bias, 'h2h_w': self._core.h2h.weight, 'h2h_b': self._core.h2h.bias,
        }

    def _train_feats(self, fc_feats, att_feats, att_masks):
        fc = self._f32(fc_feats)
        return (fc, None), None, fc.shape[0], 0


def _mha_params(d_model):
    m = nn.Module()
    m.linears = nn.ModuleList([nn.Linear(d_model, d_model) for _ in range(4)])
    return m


def _ln_params(d_model):
    m = nn.Module()
    m.a_2 = nn.Parameter(torch.ones(d_model))
    m.b_2 = nn.Parameter(torch.zeros(d_model))
    return m


def _tfm_layer(d_model, d_ff, n_sub, with_src):
    layer = nn.Module()
    layer.self_attn = _mha_params(d_model)
    if with_src:
        layer.src_attn = _mha_params(d_model)
    layer.feed_forward = nn.Module()
    layer.feed_forward.w_1 = nn.Linear(d_model, d_ff)
    layer.feed_forward.w_2 = nn.Linear(d_ff, d_model)
    layer.sublayer = nn.ModuleList()
    for _ in range(n_sub):
        sub = nn.Module()
        sub.norm = _ln_params(d_model)
        layer.sublayer.append(sub)
    return layer


class B200TransformerModel(B200CaptionModel):
    """Drop-in for captioning.models.TransformerModel.TransformerModel (TransformerModel.py:237-363): same opt fields (N_enc, N_dec,
    d_model, d_ff, num_att_heads), same state_dict keys (att_embed.0.*, model.encoder/decoder.layers.*, model.tgt_embed.0.lut.weight,
    model.tgt_embed.1.pe buffer, model.generator.proj.*).  Decoding keeps a per-layer K/V cache on the device."""

    family_name = 'transformer'
    _no_diverse = 'the decoder K/V cache and positional encoding take one position per launch, so its groups cannot be at different positions'
    # the transformer ignores fc_feats (TransformerModel.py:305-310); its positional-encoding buffer is bound but never trained
    _abi, _takes_fc, _entry = 'tfm', False, 'tfm'
    _weights_struct = _grads_struct = _lib.TfmWeights
    _bind_only = frozenset({('pe',)})
    _parallel_pass = True

    def __init__(self, opt, numeric_mode=None):
        super().__init__(opt, numeric_mode)
        import math
        self.N_enc = getattr(opt, 'N_enc', opt.num_layers)
        self.N_dec = getattr(opt, 'N_dec', opt.num_layers)
        self.d_model = getattr(opt, 'd_model', opt.input_encoding_size)
        self.d_ff = getattr(opt, 'd_ff', opt.rnn_size)
        self.h = getattr(opt, 'num_att_heads', 8)
        self.dropout = getattr(opt, 'dropout', 0.1)             # every nn.Dropout inside make_model (TransformerModel.py:240-253)
        if self.N_enc > _lib.TFM_MAX_LAYERS or self.N_dec > _lib.TFM_MAX_LAYERS:
            raise NotImplementedError('at most %d layers per stack' % _lib.TFM_MAX_LAYERS)
        V1, D = self.vocab_size + 1, self.d_model
        self.att_embed = nn.Sequential(nn.Linear(self.att_feat_size, D), nn.ReLU(), nn.Dropout(self.drop_prob_lm))
        self.model = nn.Module()
        self.model.encoder = nn.Module()
        self.model.encoder.layers = nn.ModuleList([_tfm_layer(D, self.d_ff, 2, False) for _ in range(self.N_enc)])
        self.model.encoder.norm = _ln_params(D)
        self.model.decoder = nn.Module()
        self.model.decoder.layers = nn.ModuleList([_tfm_layer(D, self.d_ff, 3, True) for _ in range(self.N_dec)])
        self.model.decoder.norm = _ln_params(D)
        emb = nn.Module()
        emb.lut = nn.Embedding(V1, D)
        pos = nn.Module()
        pe = torch.zeros(5000, D)
        position = torch.arange(0, 5000).unsqueeze(1).float()
        div_term = torch.exp(torch.arange(0, D, 2).float() * -(math.log(10000.0) / D))
        pe[:, 0::2] = torch.sin(position * div_term)
        pe[:, 1::2] = torch.cos(position * div_term)
        pos.register_buffer('pe', pe.unsqueeze(0))
        self.model.tgt_embed = nn.Sequential(emb, pos)
        self.model.generator = nn.Module()
        self.model.generator.proj = nn.Linear(D, V1)
        for p_ in self.model.parameters():        # Glorot init like make_model (TransformerModel.py:255-258)
            if p_.dim() > 1:
                nn.init.xavier_uniform_(p_)

    def _cfg(self):
        return _lib.TfmCfg(self.vocab_size, self.d_model, self.d_ff, self.h, self.N_enc, self.N_dec, self.att_feat_size, self.seq_length,
                           _lib.MODES[self.numeric_mode])

    def _slots(self):
        """[(path into capb200_tfm_weights / capb200_tfm_grads, parameter)]: path = (field,) | ('enc'|'dec', layer, field) | ('enc'|'dec', layer, attn, field)."""
        out = [(('att_embed_w',), self.att_embed[0].weight), (('att_embed_b',), self.att_embed[0].bias)]

        def layer_slots(kind, i, layer, attns, n_sub):
            for an in attns:          # q | k | v weights (and biases) back to back: one GEMM / one column reduction per triple in the engine
                lins = getattr(layer, an).linears
                for suffix, attr in (('_w', 'weight'), ('_b', 'bias')):
                    for name, lin in zip(('q', 'k', 'v'), lins):
                        out.append(((kind, i, an, name + suffix), getattr(lin, attr)))
                out.append(((kind, i, an, 'o_w'), lins[3].weight))
                out.append(((kind, i, an, 'o_b'), lins[3].bias))
            out.append(((kind, i, 'w1_w'), layer.feed_forward.w_1.weight)); out.append(((kind, i, 'w1_b'), layer.feed_forward.w_1.bias))
            out.append(((kind, i, 'w2_w'), layer.feed_forward.w_2.weight)); out.append(((kind, i, 'w2_b'), layer.feed_forward.w_2.bias))
            for j in range(n_sub):
                out.append(((kind, i, 'ln%d_a' % j), layer.sublayer[j].norm.a_2)); out.append(((kind, i, 'ln%d_b' % j), layer.sublayer[j].norm.b_2))

        for i, layer in enumerate(self.model.encoder.layers):
            layer_slots('enc', i, layer, ('self_attn',), 2)
        out += [(('enc_norm_a',), self.model.encoder.norm.a_2), (('enc_norm_b',), self.model.encoder.norm.b_2)]
        for i, layer in enumerate(self.model.decoder.layers):
            layer_slots('dec', i, layer, ('self_attn', 'src_attn'), 3)
        out += [(('dec_norm_a',), self.model.decoder.norm.a_2), (('dec_norm_b',), self.model.decoder.norm.b_2),
                (('lut',), self.model.tgt_embed[0].lut.weight), (('pe',), self.model.tgt_embed[1].pe),
                (('gen_w',), self.model.generator.proj.weight), (('gen_b',), self.model.generator.proj.bias)]
        return out

    def _grad_groups(self, named):
        late = [s for s in named if s[0].startswith(('enc', 'att_embed'))]              # encoder + att_embed finish last
        early = [s for s in named if not s[0].startswith(('enc', 'att_embed'))]
        return [early, late]

    def _rates(self, train, drop_prob=None, dropout=None):
        """drop_prob_lm (att_embed's dropout), dropout (the Transformer's own rate)"""
        if not train:
            return 0.0, 0.0
        return float(self.drop_prob_lm if drop_prob is None else drop_prob), float(self.dropout if dropout is None else dropout)

    def _xe_opts(self, spi, steps, seed, label_smoothing, upstream, rates, masks, ss_prob, tokens_used, keep_rows, row_loss):
        return _lib.TfmXeOpts(spi, seed, label_smoothing, upstream, *rates, _lib.ptr(masks), keep_rows, _lib.ptr(row_loss))

    def _scst_opts(self, sample_n, temperature, seed, upstream, baseline, rates, forced, masks, keep_rows, row_loss, sampler, rw):
        return _lib.TfmScstOpts(sample_n, temperature, seed, upstream, baseline, *rates, _lib.ptr(forced), _lib.ptr(masks), keep_rows, _lib.ptr(row_loss),
                                sampler, rw)

    @_on_device
    def xe_step(self, fc_feats, att_feats, labels, masks, label_smoothing=0.0, drop_prob=None, seed=None, upstream=1.0, dropout=None, att_masks=None,
                keep_rows=0):
        """One cross-entropy step of the Transformer on the device (capb200_tfm_xe_step): the teacher-forced pass over every position
        (TransformerModel.py:340-348), LanguageModelCriterion / LabelSmoothing, backward through decoder and encoder.  ``drop_prob`` is
        att_embed's dropout (drop_prob_lm), ``dropout`` the Transformer's own rate.  self.ss_prob is ignored, as in the reference:
        TransformerModel._forward is one parallel pass with no scheduled-sampling branch.  Result as B200UpDownModel.xe_step."""
        return self._xe_step(fc_feats, att_feats, labels, masks, self._rates(True, drop_prob, dropout), label_smoothing, seed, upstream, att_masks,
                             keep_rows)

    @_on_device
    def scst_step(self, fc_feats, att_feats, gts, table, sample_n, temperature=1.0, drop_prob=None, seed=None, upstream=1.0, baseline='greedy', dropout=None,
                  forced_tokens=None, att_masks=None, keep_rows=0, reward_weights=None, sample_method='sample', baseline_method='greedy',
                  forced_baseline=None):
        """One self-critical step of the Transformer on the device (capb200_tfm_scst_step): eval-mode greedy baseline (or leave-one-out),
        train-mode samples drawn position by position on the K/V tape, CIDEr-D (or weighted, ``reward_weights``) reward, RewardCriterion,
        batched backward.  ``sample_method`` / ``baseline_method`` / ``forced_baseline`` and the result as B200UpDownModel.scst_step."""
        return self._scst_step(fc_feats, att_feats, gts, table, sample_n, self._rates(True, drop_prob, dropout), temperature, seed, upstream, baseline,
                               forced_tokens, att_masks, keep_rows, reward_weights, sample_method, baseline_method, forced_baseline)


class B200AoAModel(B200CaptionModel):
    """Drop-in for captioning.models.AoAModel.AoAModel in the configs/aoa.yml configuration (refine=1, refine_aoa=1, use_ff=0,
    decoder_type='AoA', use_multi_head=2, multi_head_scale=1, mean_feats=1): same state_dict keys (no fc_embed), same surfaces."""

    family = _lib.FAMILY_AOA
    family_name = 'aoa'
    _abi, _takes_fc, _entry = 'aoa', False, 'aoa'
    _weights_struct = _grads_struct = _lib.AoaWeights

    def __init__(self, opt, numeric_mode=None):
        super().__init__(opt, numeric_mode)
        need = dict(refine=1, refine_aoa=1, use_ff=0, decoder_type='AoA', use_multi_head=2, multi_head_scale=1)
        for k, v in need.items():
            if getattr(opt, k, v) != v:
                raise NotImplementedError('AoA option %s=%r is outside the configs/aoa.yml configuration the engine implements' % (k, getattr(opt, k)))
        if not getattr(opt, 'mean_feats', 1):
            raise NotImplementedError('mean_feats=0 is outside the configs/aoa.yml configuration')
        if getattr(opt, 'out_res', 0):
            raise NotImplementedError('out_res is outside the configs/aoa.yml configuration')
        self.num_layers = 2
        self.num_heads = opt.num_heads
        self.dropout_aoa = getattr(opt, 'dropout_aoa', 0.3)          # AoAModel.py:117
        self.ctx_drop = getattr(opt, 'ctx_drop', 0)                  # AoAModel.py:134
        H, E, V1 = self.rnn_size, self.input_encoding_size, self.vocab_size + 1
        self.embed = nn.Sequential(nn.Embedding(V1, E), nn.ReLU(), nn.Dropout(self.drop_prob_lm))
        self.att_embed = nn.Sequential(nn.Linear(self.att_feat_size, H), nn.ReLU(), nn.Dropout(self.drop_prob_lm))
        self.logit = self._make_logit()
        self.ctx2att = nn.Linear(H, 2 * H)
        self.refiner = nn.Module()
        self.refiner.layers = nn.ModuleList()
        for _ in range(_lib.AOA_REFINER_LAYERS):
            layer = nn.Module()
            layer.self_attn = nn.Module()
            layer.self_attn.linears = nn.ModuleList([nn.Linear(H, H) for _ in range(3)])
            layer.self_attn.aoa_layer = nn.Sequential(nn.Linear(2 * H, 2 * H), nn.GLU())
            sub = nn.Module()
            sub.norm = _ln_params(H)
            layer.sublayer = nn.ModuleList([sub])
            self.refiner.layers.append(layer)
        self.refiner.norm = _ln_params(H)
        self.core = nn.Module()
        self.core.att_lstm = nn.LSTMCell(E + H, H)
        self.core.att2ctx = nn.Sequential(nn.Linear(2 * H, 2 * H), nn.GLU())
        self.core.attention = nn.Module()
        self.core.attention.norm = _ln_params(H)
        self.core.attention.linears = nn.ModuleList([nn.Linear(H, H)])

    def _cfg(self):
        return _lib.AoaCfg(self.vocab_size, self.input_encoding_size, self.rnn_size, self.num_heads, self.att_feat_size, self.seq_length,
                           _lib.MODES[self.numeric_mode])

    def _slots(self):
        """(field path in capb200_aoa_weights / capb200_aoa_grads, parameter) pairs."""
        out = [(('embed',), self.embed[0].weight), (('att_embed_w',), self.att_embed[0].weight), (('att_embed_b',), self.att_embed[0].bias)]
        for i, layer in enumerate(self.refiner.layers):
            for name, lin in zip(('q', 'k', 'v'), layer.self_attn.linears):
                out += [(('refiner', i, name + '_w'), lin.weight), (('refiner', i, name + '_b'), lin.bias)]
            out += [(('refiner', i, 'aoa_w'), layer.self_attn.aoa_layer[0].weight), (('refiner', i, 'aoa_b'), layer.self_attn.aoa_layer[0].bias),
                    (('refiner', i, 'ln_a'), layer.sublayer[0].norm.a_2), (('refiner', i, 'ln_b'), layer.sublayer[0].norm.b_2)]
        c = self.core
        out += [(('refiner_norm_a',), self.refiner.norm.a_2), (('refiner_norm_b',), self.refiner.norm.b_2),
                (('ctx2att_w',), self.ctx2att.weight), (('ctx2att_b',), self.ctx2att.bias),
                (('att_lstm_w_ih',), c.att_lstm.weight_ih), (('att_lstm_w_hh',), c.att_lstm.weight_hh),
                (('att_lstm_b_ih',), c.att_lstm.bias_ih), (('att_lstm_b_hh',), c.att_lstm.bias_hh),
                (('attn_norm_a',), c.attention.norm.a_2), (('attn_norm_b',), c.attention.norm.b_2),
                (('attn_q_w',), c.attention.linears[0].weight), (('attn_q_b',), c.attention.linears[0].bias),
                (('att2ctx_w',), c.att2ctx[0].weight), (('att2ctx_b',), c.att2ctx[0].bias),
                (('logit_w',), self._vocab_logit.weight), (('logit_b',), self._vocab_logit.bias)]
        return out

    def _grad_groups(self, named):
        slots = dict(named)
        pick = lambda names: [(n, slots[n]) for n in names]
        groups = [pick(['logit_w', 'logit_b'] + [n for n, _ in self._head_named()]),
                  pick(['att2ctx_w', 'att2ctx_b', 'attn_q_w', 'attn_q_b', 'att_lstm_w_ih', 'att_lstm_w_hh', 'att_lstm_b_ih', 'att_lstm_b_hh', 'attn_norm_a',
                        'attn_norm_b', 'embed']),
                  pick(['ctx2att_w', 'ctx2att_b', 'refiner_norm_a', 'refiner_norm_b'])]
        for l in reversed(range(_lib.AOA_REFINER_LAYERS)):
            # q | k | v weights (and biases) back to back: the engine then writes each triple with one GEMM / one column reduction
            groups.append(pick(['refiner/%d/%s' % (l, f) for f in ('q_w', 'k_w', 'v_w', 'q_b', 'k_b', 'v_b', 'aoa_w', 'aoa_b', 'ln_a', 'ln_b')]))
        groups.append(pick(['att_embed_w', 'att_embed_b']))
        assert sum(len(g) for g in groups) == len(slots)
        return groups

    def _rates(self, train, drop_prob=None, drop_attn=0.1, drop_aoa=None, drop_sublayer=0.1, ctx_drop=None):
        """drop_prob_lm, drop_attn, drop_aoa, drop_sublayer, ctx_drop"""
        if not train:
            return 0.0, 0.0, 0.0, 0.0, 0
        return (float(self.drop_prob_lm if drop_prob is None else drop_prob), float(drop_attn), float(self.dropout_aoa if drop_aoa is None else drop_aoa),
                float(drop_sublayer), int(self.ctx_drop if ctx_drop is None else ctx_drop))

    def _xe_opts(self, spi, steps, seed, label_smoothing, upstream, rates, masks, ss_prob, tokens_used, keep_rows, row_loss):
        return _lib.AoaXeOpts(spi, steps, seed, label_smoothing, upstream, *rates, _lib.ptr(masks), ss_prob, _lib.ptr(tokens_used), keep_rows,
                              _lib.ptr(row_loss))

    def _scst_opts(self, sample_n, temperature, seed, upstream, baseline, rates, forced, masks, keep_rows, row_loss, sampler, rw):
        return _lib.AoaScstOpts(sample_n, temperature, seed, upstream, baseline, *rates, _lib.ptr(forced), _lib.ptr(masks), keep_rows, _lib.ptr(row_loss),
                                sampler, rw)

    @_on_device
    def scst_step(self, fc_feats, att_feats, gts, table, sample_n, temperature=1.0, drop_prob=None, seed=None, upstream=1.0, baseline='greedy',
                  drop_attn=0.1, drop_aoa=None, drop_sublayer=0.1, ctx_drop=None, forced_tokens=None, att_masks=None, keep_rows=0, reward_weights=None,
                  sample_method='sample', baseline_method='greedy', forced_baseline=None):
        """One self-critical step of AoANet on the device (capb200_aoa_scst_step): eval-mode greedy baseline (or the leave-one-out baseline of
        'new_self_critical'), train-mode samples with every dropout site of AoAModel.py active, CIDEr-D reward, RewardCriterion, BPTT through
        the decoder and the six refiner layers.  ``fc_feats`` is unused (mean_feats=1).  ``reward_weights``, ``sample_method``,
        ``baseline_method`` and ``forced_baseline`` as in B200UpDownModel.scst_step.
        Returns the dict of B200UpDownModel.scst_step."""
        return self._scst_step(fc_feats, att_feats, gts, table, sample_n, self._rates(True, drop_prob, drop_attn, drop_aoa, drop_sublayer, ctx_drop),
                               temperature, seed, upstream, baseline, forced_tokens, att_masks, keep_rows, reward_weights, sample_method, baseline_method,
                               forced_baseline)

    @_on_device
    def xe_step(self, fc_feats, att_feats, labels, masks, label_smoothing=0.0, drop_prob=None, seed=None, upstream=1.0, drop_attn=0.1, drop_aoa=None,
                drop_sublayer=0.1, ctx_drop=None, att_masks=None, keep_rows=0):
        """One cross-entropy step of AoANet on the device (capb200_aoa_xe_step); arguments and result as B200UpDownModel.xe_step."""
        return self._xe_step(fc_feats, att_feats, labels, masks, self._rates(True, drop_prob, drop_attn, drop_aoa, drop_sublayer, ctx_drop),
                             label_smoothing, seed, upstream, att_masks, keep_rows)


class B200AttEnsemble(B200CaptionModel):
    """Drop-in for captioning.models.AttEnsemble.AttEnsemble (test-time ensemble, tools/eval_ensemble.py): ``models`` are engine models of
    the UpDown, Att2in2, NewFC and AoANet families (any mix), ``weights`` a buffer that defaults to ``[1.0] * K``; vocab_size, seq_length and
    bad_endings_ix come from ``models[0]``.  Every step mixes the members' word distributions into log(sum_k softmax(z_k) w_k / sum_k w_k)
    (AttEnsemble.get_logprobs_state) on the device and decodes from that row: greedy and sampling ``forward(fc, att, masks, opt,
    mode='sample')``, beam search (with ``done_beams``) and teacher forcing ``forward(fc, att, seq, masks)``, with the reference's shapes.

    AttEnsemble skips AttModel.__init__, so the reference class lacks bos_idx / eos_idx / pad_idx / unk_idx / vocab, which its decode loops
    and eval_split read; this mirror takes them from ``models[0]`` as well.  Eval only: diverse beam search, output_logsoftmax=0,
    Transformer members and training raise NotImplementedError."""

    family_name = 'AttEnsemble'
    _abi = 'ensemble'
    _no_diverse = 'an ensemble runs group_size 1 only'

    def __init__(self, models, weights=None):
        nn.Module.__init__(self)
        models = list(models)
        if not 1 <= len(models) <= _lib.ENSEMBLE_MAX_MEMBERS:
            raise ValueError('an ensemble has 1..%d members (got %d)' % (_lib.ENSEMBLE_MAX_MEMBERS, len(models)))
        for m in models:
            if not isinstance(m, (B200UpDownModel, B200NewFCModel, B200AoAModel)):       # B200Att2in2Model is a B200UpDownModel
                raise NotImplementedError('ensemble members are UpDown, Att2in2, NewFC or AoANet engine models (got %s)' % type(m).__name__)
        m0 = models[0]
        for m in models[1:]:
            if m.vocab_size != m0.vocab_size or m.seq_length != m0.seq_length:
                raise ValueError('every member needs the first member\'s vocab_size and seq_length (%d, %d); got (%d, %d)'
                                 % (m0.vocab_size, m0.seq_length, m.vocab_size, m.seq_length))
        weights = weights or [1.0] * len(models)
        if len(weights) != len(models):
            raise ValueError('one weight per member (%d members, %d weights)' % (len(models), len(weights)))
        if any(not float(w) >= 0.0 or float(w) == float('inf') for w in weights) or not sum(float(w) for w in weights) > 0.0:
            raise ValueError('ensemble weights must be finite, >= 0 and not all zero (got %r)' % (list(weights),))
        self.models = nn.ModuleList(models)
        self.vocab_size, self.seq_length, self.bad_endings_ix = m0.vocab_size, m0.seq_length, m0.bad_endings_ix
        self.vocab, self.bos_idx, self.eos_idx, self.pad_idx, self.unk_idx = m0.vocab, m0.bos_idx, m0.eos_idx, m0.pad_idx, m0.unk_idx
        self.numeric_mode = m0.numeric_mode
        self.ss_prob = 0
        self.register_buffer('weights', torch.tensor(weights))
        self.done_beams = []
        self._store = _EngineStore(self)

    def _ensure_engine(self, device):
        devices = {p.device for m in self.models for p in m.parameters()}
        if devices != {device}:
            raise ValueError('every ensemble member must live on the device of the inputs (%s); members are on %s' % (device, sorted(map(str, devices))))
        if any(m.seq_length != self.seq_length or m.vocab_size != self.vocab_size for m in self.models):
            raise ValueError('the ensemble decodes with its members\' vocab_size and seq_length: set max_length on every member, not on the ensemble')
        weights = [float(w) for w in self.weights.tolist()]
        if any(not w >= 0.0 or w == float('inf') for w in weights) or not sum(weights) > 0.0:
            raise ValueError('ensemble weights must be finite, >= 0 and not all zero (got %r)' % weights)
        for m in self.models:
            m._ensure_engine(device)
        members = (_lib.EnsembleMember * len(self.models))()
        for k, (m, w) in enumerate(zip(self.models, weights)):
            members[k].family = m.family
            members[k].engine, members[k].weight = m._engine, w
        lib = self._enter_device(device)
        if self._engine is None:
            self._engine = lib.capb200_ensemble_create()
        self._members = members
        return lib

    def _call_sample(self, lib, fc, att, masks, B, R, so, tok, ld_tok, seq, logprobs):
        return lib.capb200_ensemble_decode_sample(self._engine, self._members, len(self._members), _lib.ptr(fc), _lib.ptr(att), _lib.ptr(masks), B, R,
                                                  ctypes.byref(so), _lib.ptr(tok), ld_tok, _lib.ptr(seq), _lib.ptr(logprobs), None, _lib.current_stream())

    def _call_beam(self, lib, fc, att, masks, B, R, bo, seq, logprobs, d_seq, d_len, d_p, d_raw):
        return lib.capb200_ensemble_decode_beam(self._engine, self._members, len(self._members), _lib.ptr(fc), _lib.ptr(att), _lib.ptr(masks), B, R,
                                                ctypes.byref(bo), _lib.ptr(seq), _lib.ptr(logprobs), _lib.ptr(d_seq), _lib.ptr(d_len), _lib.ptr(d_p),
                                                _lib.ptr(d_raw), _lib.current_stream())

    def _call_record(self, lib, image, rank, dst):
        return lib.capb200_ensemble_beam_record_logprobs(self._engine, image, rank, _lib.ptr(dst), _lib.current_stream())

    def scst_step(self, *args, **kwargs):
        raise NotImplementedError('an ensemble is a test-time model: train its members')

    def xe_step(self, *args, **kwargs):
        raise NotImplementedError('an ensemble is a test-time model: train its members')


def setup(opt, numeric_mode=None):
    """Factory with the contract of captioning.models.setup (captioning/models/__init__.py:20-73) for the families on the
    engine hot path."""
    name = opt.caption_model
    if name in ('topdown', 'updown'):
        return B200UpDownModel(opt, numeric_mode)
    if name == 'newfc':
        return B200NewFCModel(opt, numeric_mode)
    if name == 'att2in2':
        return B200Att2in2Model(opt, numeric_mode)
    if name == 'aoa':
        return B200AoAModel(opt, numeric_mode)
    if name == 'transformer':
        if getattr(opt, 'cached_transformer', False):
            raise NotImplementedError('cachedTransformer is a reference-side variant; the engine always caches K/V')
        return B200TransformerModel(opt, numeric_mode)
    raise NotImplementedError('caption_model %r is not on the engine decode path yet (SURVEY.md section 8)' % name)
