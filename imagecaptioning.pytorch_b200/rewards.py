"""Device-side mirror of captioning/utils/rewards.py for the SCST inner loop.

    init_scorer(cached_tokens)                                   rewards.py:25-31
    get_self_critical_reward(greedy_res, data_gts, gen_result, opt)   rewards.py:41-81
    get_scores(data_gts, gen_result, opt)                             rewards.py:83-114
    get_self_cider_scores(data_gts, gen_result, opt)                  rewards.py:116-138

The reference moves both id tensors to the host, formats every id as a string and walks Python dicts; here the ids
never leave the GPU: n-gram extraction, the document-frequency lookup (open-addressing hash table built once from the
``scripts/prepro_ngrams.py`` pickle), the clipped tf-idf cosine and the self-critical difference run in csrc/reward.cu.

The reward is ``cider_reward_weight * CIDEr-D + bleu_reward_weight * BLEU-4`` (opts.py:169-172), a term computed only when its weight is
> 0.  The BLEU-4 term is the per-sentence BLEU-4 of coco-caption's Bleu(4) scorer (closest reference length), also computed on the device.
With ``bleu_reward_weight <= 0`` the functions below take the CIDEr-D-only path they always took.
"""
from __future__ import annotations

import ctypes
import os
import pickle
import threading
from typing import Dict, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib


class CiderDTable:
    """Owns the device hash tables n-gram -> idf (capb200_cider_table), one per GPU, built lazily on the device that asks (under
    nn.DataParallel every replica scores its shard on its own GPU)."""

    def __init__(self, document_frequency: Dict[Tuple, float], ref_len: float, device=None):
        n = len(document_frequency)
        keys = np.full((max(n, 1), 4), -1, dtype=np.int32)
        vals = np.zeros((max(n, 1),), dtype=np.float64)
        for i, (k, v) in enumerate(document_frequency.items()):
            keys[i, :len(k)] = [int(t) for t in k]        # pickle keys are tuples of id strings (prepro_ngrams.py:42-45)
            vals[i] = float(v)
        self._keys, self._vals = keys, vals
        self.ref_len = float(ref_len)
        self.entries = n
        self._handles = {}
        self._lock = threading.Lock()
        self.device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        self._handle(self.device.index if self.device.index is not None else torch.cuda.current_device())

    def _handle(self, index: int):
        with self._lock:
            h = self._handles.get(index)
            if h is None:
                lib = _lib.load()
                with torch.cuda.device(index):
                    h = lib.capb200_cider_table_create(self._keys.ctypes.data, self._vals.ctypes.data, self.entries, self.ref_len, _lib.current_stream())
                if not h:
                    raise RuntimeError('capb200 cider_table_create failed: %s' % lib.capb200_last_error().decode())
                self._handles[index] = h
            return h

    @property
    def _h(self):
        """Handle of the table on the calling thread's current CUDA device."""
        return self._handle(torch.cuda.current_device())

    def handle_for(self, refs: torch.Tensor):
        """The handle a reward call over the packed reference rows `refs` [n_refs, L] passes to the C ABI."""
        return self._h

    @classmethod
    def from_pickle(cls, path: str, device=None):
        with open(path, 'rb') as f:
            pk = pickle.load(f, encoding='latin1')
        return cls(pk['document_frequency'], pk['ref_len'], device)

    def __del__(self):
        try:
            for h in self._handles.values():
                _lib.load().capb200_cider_table_destroy(h)
            self._handles = {}
        except Exception:
            pass


class CorpusCiderDTable(CiderDTable):
    """CiderD(df='corpus') (ciderD_scorer.py:143-147, 182-186, 210-216): no pickle; every reward call rebuilds the document frequencies on
    the device from its own references (capb200_cider_corpus_table_create).  df counts the scored hypotheses whose image has the n-gram
    among its references, ref_len = log(number of hypotheses): an SCST call counts each image n + 1 times, get_scores n times."""

    def __init__(self, device=None):
        self.ref_len = None
        self.entries = 0
        self._handles = {}
        self._lock = threading.Lock()
        self.device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        self._handle(self.device.index if self.device.index is not None else torch.cuda.current_device())

    def _handle(self, index: int):
        with self._lock:
            h = self._handles.get(index)
            if h is None:
                lib = _lib.load()
                with torch.cuda.device(index):
                    h = lib.capb200_cider_corpus_table_create()
                if not h:
                    raise RuntimeError('capb200 cider_corpus_table_create failed: %s' % lib.capb200_last_error().decode())
                self._handles[index] = h
            return h

    def handle_for(self, refs: torch.Tensor):
        h = self._h
        _lib.check(_lib.load().capb200_cider_table_reserve(h, int(refs.shape[0]), int(refs.shape[1])), 'cider_table_reserve')
        return h


CiderD_scorer: Optional[CiderDTable] = None


def init_scorer(cached_tokens, device=None):
    """Same contract as the reference: ``cached_tokens`` names ``data/<cached_tokens>.p`` relative to the cwd
    (ciderD_scorer.py:109), and ``'corpus'`` takes the document frequencies from the references of each call (no file); an existing path
    or an already built CiderDTable is accepted too.  Idempotent."""
    global CiderD_scorer
    if CiderD_scorer is not None:
        return CiderD_scorer
    if isinstance(cached_tokens, CiderDTable):
        CiderD_scorer = cached_tokens
    elif cached_tokens == 'corpus':
        CiderD_scorer = CorpusCiderDTable(device)
    else:
        path = cached_tokens if os.path.exists(str(cached_tokens)) else os.path.join('data', str(cached_tokens) + '.p')
        CiderD_scorer = CiderDTable.from_pickle(path, device)
    return CiderD_scorer


def reset_scorer():
    global CiderD_scorer
    CiderD_scorer = None


class _Staging:
    """Per-step reference upload: round-robin PINNED host blocks (a block is reused only after the copy that read it has completed) feeding ONE
    device buffer per GPU -- the padded reference rows and the offsets travel in a single asynchronous H2D copy, and the device addresses stay
    the same from step to step (copies and the kernels that read them are ordered on the stream), which is what lets the engine replay the
    SCST step as a CUDA graph."""
    SLOTS = 4

    def __init__(self):
        self.host = {}
        self.dev = {}
        self.turn = 0

    def upload(self, host_rows: np.ndarray, offs: np.ndarray, device):
        dev = torch.device(device)
        idx = dev.index if dev.index is not None else torch.cuda.current_device()
        head = (offs.size + 1023) // 1024 * 1024          # offsets first, in a fixed-size head: both device addresses are independent of the row count
        n = head + host_rows.size
        cap = max(n, 1 << 14)
        key = (idx, self.turn % self.SLOTS)
        self.turn += 1
        slot = self.host.get(key)
        if slot is None or slot[0].numel() < n:
            slot = [torch.empty(cap, dtype=torch.int32).pin_memory(), None]
            self.host[key] = slot
        pinned, ev = slot
        if ev is not None:
            ev.synchronize()
        devbuf = self.dev.get(idx)
        if devbuf is None or devbuf.numel() < n:
            devbuf = torch.empty(cap, dtype=torch.int32, device=dev)
            self.dev[idx] = devbuf
        flat = pinned.numpy()
        flat[:offs.size] = offs
        flat[head:n] = host_rows.reshape(-1)
        devbuf[:n].copy_(pinned[:n], non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(dev))
        slot[1] = ev
        return devbuf[head:n].view(host_rows.shape), devbuf[:offs.size]


_staging = _Staging()


def pack_references(data_gts: Sequence, device) -> Tuple[torch.Tensor, torch.Tensor, int]:
    """list[B] of int arrays [n_refs_i, L] (dataloader.py:213) -> (refs int32 [total, L], offsets int32 [B+1], L) on the device.
    The returned tensors are views of the device staging buffer, overwritten by the next upload (in stream order): consume them in the step
    they were packed for."""
    L = max(int(np.asarray(g).shape[1]) for g in data_gts)
    total = sum(int(np.asarray(g).shape[0]) for g in data_gts)
    rows = np.zeros((total, L), dtype=np.int32)
    offs = np.zeros(len(data_gts) + 1, dtype=np.int32)
    at = 0
    for i, g in enumerate(data_gts):
        g = np.asarray(g)
        rows[at:at + g.shape[0], :g.shape[1]] = g
        at += g.shape[0]
        offs[i + 1] = at
    if torch.device(device).type != 'cuda':
        return torch.from_numpy(rows), torch.from_numpy(offs), L
    refs, offsets = _staging.upload(rows, offs, device)
    return refs, offsets, L


def cider_scores_and_reward(greedy_res: torch.Tensor, data_gts: Sequence, gen_result: torch.Tensor, table: Optional[CiderDTable] = None):
    table = table or CiderD_scorer
    if table is None:
        raise RuntimeError('init_scorer(cached_tokens) must be called before the SCST reward (tools/train.py:150-152)')
    dev = gen_result.device
    if dev.type != 'cuda':
        raise RuntimeError('capb200: the reward kernel runs on CUDA tensors only')
    B = len(data_gts)
    S, T = gen_result.shape
    assert greedy_res.shape[0] == B and S % B == 0
    sampled = gen_result.detach().to(torch.long).contiguous()
    greedy = greedy_res.detach().to(torch.long).contiguous()
    refs, offsets, L = pack_references(data_gts, dev)
    scores = torch.empty(S + B, dtype=torch.float64, device=dev)
    reward = torch.empty(S, T, dtype=torch.float32, device=dev)
    lib = _lib.load()
    _lib.check(lib.capb200_self_critical_reward(table.handle_for(refs), _lib.ptr(sampled), S, _lib.ptr(greedy), B, T, _lib.ptr(refs), _lib.ptr(offsets), L,
                                                _lib.ptr(scores), _lib.ptr(reward), _lib.current_stream()), 'self_critical_reward')
    return scores, reward


def reward_weights(opt) -> Tuple[float, float]:
    """(cider_reward_weight, bleu_reward_weight) of a training opt, with the reference's defaults (opts.py:169-172)."""
    return float(getattr(opt, 'cider_reward_weight', 1)), float(getattr(opt, 'bleu_reward_weight', 0))


def weights_struct(weights, data_gts: Sequence) -> Optional[_lib.RewardWeights]:
    """capb200_reward_weights for (cider, bleu) weights, or None (the CIDEr-D reward) for None.  With the BLEU term on, every image needs
    at least one reference (the reference asserts it, bleu.py): refused here, before any device work."""
    if weights is None:
        return None
    wc, wb = (float(w) for w in weights)
    if not (np.isfinite(wc) and np.isfinite(wb)):
        raise ValueError('reward weights must be finite')
    if wb > 0 and any(int(np.asarray(g).shape[0]) == 0 for g in data_gts):
        raise ValueError('the BLEU-4 reward needs at least one reference per image')
    return _lib.RewardWeights(wc, wb)


def _check_scorer(table, weights):
    table = table or CiderD_scorer
    if table is None and float(weights[0]) > 0:
        raise RuntimeError('init_scorer(cached_tokens) must be called before the SCST reward (tools/train.py:150-152)')
    return table


def weighted_scores(data_gts: Sequence, gen_result: torch.Tensor, weights, greedy_res: Optional[torch.Tensor] = None,
                    table: Optional[CiderDTable] = None, with_reward: bool = False):
    """``weights[0] * CIDEr-D + weights[1] * BLEU-4`` of every sampled caption -- and, with ``greedy_res``, of every greedy caption after
    them -- as float64 [S (+B)] (capb200_weighted_reward).  with_reward: also the fp32 reward [S, T], the self-critical difference with
    ``greedy_res``, else the leave-one-out reward of 'new_self_critical'."""
    w = weights_struct(weights, data_gts)
    table = _check_scorer(table, weights)
    dev = gen_result.device
    if dev.type != 'cuda':
        raise RuntimeError('capb200: the reward kernel runs on CUDA tensors only')
    B = len(data_gts)
    S, T = gen_result.shape
    assert S % B == 0 and (greedy_res is None or greedy_res.shape[0] == B)
    sampled = gen_result.detach().to(torch.long).contiguous()
    greedy = None if greedy_res is None else greedy_res.detach().to(torch.long).contiguous()
    refs, offsets, L = pack_references(data_gts, dev)
    hyps = S + (0 if greedy is None else B)
    scores = torch.empty(hyps, dtype=torch.float64, device=dev)
    bleu = torch.empty(hyps, dtype=torch.float64, device=dev)
    reward = torch.empty(S, T, dtype=torch.float32, device=dev) if with_reward else None
    lib = _lib.load()
    _lib.check(lib.capb200_weighted_reward(table.handle_for(refs) if table is not None else None, ctypes.byref(w), _lib.ptr(sampled), S, _lib.ptr(greedy), B, T,
                                           _lib.ptr(refs), _lib.ptr(offsets), L, _lib.ptr(scores), _lib.ptr(bleu), _lib.ptr(reward),
                                           _lib.current_stream()), 'weighted_reward')
    return (scores, reward) if with_reward else scores


def bleu_scores(data_gts: Sequence, gen_result: torch.Tensor, greedy_res: Optional[torch.Tensor] = None):
    """Per-sentence BLEU-4 (Bleu(4).compute_score(...)[1][3], closest reference length) of every sampled caption against its image's
    references -- and, with ``greedy_res``, of every greedy caption after them: float64 [S (+B)] on the device (capb200_bleu4_scores)."""
    weights_struct((0.0, 1.0), data_gts)
    dev = gen_result.device
    if dev.type != 'cuda':
        raise RuntimeError('capb200: the reward kernel runs on CUDA tensors only')
    B = len(data_gts)
    S, T = gen_result.shape
    assert S % B == 0 and (greedy_res is None or greedy_res.shape[0] == B)
    sampled = gen_result.detach().to(torch.long).contiguous()
    greedy = None if greedy_res is None else greedy_res.detach().to(torch.long).contiguous()
    refs, offsets, L = pack_references(data_gts, dev)
    scores = torch.empty(S + (0 if greedy is None else B), dtype=torch.float64, device=dev)
    _lib.check(_lib.load().capb200_bleu4_scores(_lib.ptr(sampled), S, _lib.ptr(greedy), B, T, _lib.ptr(refs), _lib.ptr(offsets), L, _lib.ptr(scores),
                                                _lib.current_stream()), 'bleu4_scores')
    return scores


def get_self_critical_reward(greedy_res, data_gts, gen_result, opt):
    """reward[i*n+j, :] = score(sample j of image i) - score(greedy of image i), score = cider_reward_weight * CIDEr-D + bleu_reward_weight
    * BLEU-4, as a device fp32 tensor [S, T] (the reference returns the same values as a host float64 array that LossWrapper immediately
    moves back to the GPU)."""
    wc, wb = reward_weights(opt)
    if wb > 0:
        _, reward = weighted_scores(data_gts, gen_result, (wc, wb), greedy_res=greedy_res, with_reward=True)
        return reward
    w = wc
    _, reward = cider_scores_and_reward(greedy_res, data_gts, gen_result)
    return reward if w == 1.0 else reward * w


def cider_scores(data_gts: Sequence, gen_result: torch.Tensor, table: Optional[CiderDTable] = None, with_reward: bool = False):
    """CIDEr-D of every sampled caption (float64 [S]) and, optionally, the leave-one-out reward [S, T] (capb200_cider_scores)."""
    table = table or CiderD_scorer
    if table is None:
        raise RuntimeError('init_scorer(cached_tokens) must be called before the structure-loss scores (tools/train.py:150-152)')
    dev = gen_result.device
    if dev.type != 'cuda':
        raise RuntimeError('capb200: the reward kernel runs on CUDA tensors only')
    B = len(data_gts)
    S, T = gen_result.shape
    assert S % B == 0
    sampled = gen_result.detach().to(torch.long).contiguous()
    refs, offsets, L = pack_references(data_gts, dev)
    scores = torch.empty(S, dtype=torch.float64, device=dev)
    reward = torch.empty(S, T, dtype=torch.float32, device=dev) if with_reward else None
    lib = _lib.load()
    _lib.check(lib.capb200_cider_scores(table.handle_for(refs), _lib.ptr(sampled), S, B, T, _lib.ptr(refs), _lib.ptr(offsets), L, _lib.ptr(scores),
                                        _lib.ptr(reward) if with_reward else None, _lib.current_stream()), 'cider_scores')
    return (scores, reward) if with_reward else scores


def get_scores(data_gts, gen_result, opt):
    """rewards.py:83-114: ``cider_reward_weight * CIDEr-D + bleu_reward_weight * BLEU-4`` per sampled caption, float64 [S] on the device
    (the reference returns the same values as a host numpy array)."""
    wc, wb = reward_weights(opt)
    if wb > 0:
        return weighted_scores(data_gts, gen_result, (wc, wb))
    w = wc
    scores = cider_scores(data_gts, gen_result)
    return scores if w == 1.0 else scores * w


def _self_cider_table(table: Optional[CiderDTable]) -> CiderDTable:
    table = table or CiderD_scorer
    if table is None:
        raise RuntimeError('init_scorer(cached_tokens) must be called before the self-CIDEr scores (tools/train.py:150-152)')
    if isinstance(table, CorpusCiderDTable):
        raise NotImplementedError("self-CIDEr needs document frequencies with a reference length; a corpus table (init_scorer('corpus')) has "
                                  "none until a CIDEr-D score has been computed, and the reference fails its assert there too")
    return table


def check_caption_sets(rows: int, n: int, T: int) -> int:
    """Number of images of ``rows`` captions in sets of ``n``; raises ValueError for the shapes the diversity kernels refuse.  Those keep
    captions of at most 64 tokens, while the CIDEr-D / BLEU-4 rewards take up to 256 (CAPB200_MAX_SEQ_LENGTH)."""
    if n < 2:
        raise ValueError('diversity needs at least 2 captions per image (log(n) = 0 below that), got %d' % n)
    if n > 32:
        raise ValueError('at most 32 captions per image, got %d' % n)
    if rows % n:
        raise ValueError('%d captions do not split into sets of %d' % (rows, n))
    if T < 1 or T > 64:
        raise ValueError('caption length between 1 and 64 tokens, got %d' % T)
    return rows // n


def self_cider(seqs: torch.Tensor, n: int, table: Optional[CiderDTable] = None, with_eos: bool = True):
    """(matrices float64 [B, n, n], scores float64 [B]) on the device (capb200_self_cider): each image's n x n self-CIDEr matrix
    (CiderScorer.my_get_self_cider) and its eigenvalue diversity.  with_eos keeps each caption through its first 0, as array_to_str does;
    without it the caption stops before the 0, as the decoded words do."""
    rows, T = seqs.shape
    B = check_caption_sets(int(rows), int(n), int(T))
    table = _self_cider_table(table)
    dev = seqs.device
    if dev.type != 'cuda':
        raise RuntimeError('capb200: the diversity kernels run on CUDA tensors only')
    ids = seqs.detach().to(torch.long).contiguous()
    out = torch.empty(B * n * n + B, dtype=torch.float64, device=dev)
    _lib.check(_lib.load().capb200_self_cider(table._h, _lib.ptr(ids), B, n, T, 1 if with_eos else 0, _lib.ptr(out), _lib.ptr(out[B * n * n:]),
                                              _lib.current_stream()), 'self_cider')
    return out[:B * n * n].view(B, n, n), out[B * n * n:]


def get_self_cider_scores(data_gts, gen_result, opt):
    """rewards.py:116-138: the eigenvalue diversity of each image's self-CIDEr matrix, float64 [len(data_gts)] on the device (the
    reference returns the same values as a host numpy array, as get_scores does).  Captions are cut through their first 0, as array_to_str
    writes them; the document frequencies and ref_len are those init_scorer loaded (the reference's Cider(df=cached_tokens) reads the
    same pickle).  An n-gram missing from the table counts as df 0 where the reference's plain dict raises KeyError."""
    rows = int(gen_result.shape[0])
    n = rows // max(len(data_gts), 1)
    check_caption_sets(rows, n, int(gen_result.shape[1]))
    return self_cider(gen_result, n, with_eos=True)[1]
