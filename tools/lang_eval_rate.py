"""Time of language evaluation on the device: coco-caption's BLEU-1..4, ROUGE-L and CIDEr of a validation split (csrc/coco_eval.cu).

    python tools/lang_eval_rate.py [--images 5000] [--refs 5] [--steps 5] [--windows 7]

--images images x --refs references, captions and references of 8-16 tokens (T = 16, V = 9487, seeded ids from a per-image pool of
words, so captions share n-grams with their references).  Two numbers, each the median over --windows windows of --steps calls:
* kernels: the capb200_coco_scores call alone on packed references, between CUDA events;
* coco_scores: eval_multi.coco_scores end to end -- reference packing and upload, the kernels, the one read-back and the result dicts.
Prints one JSON line with the device name and power limit read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tools'))

from dbs_rate import device_info                  # noqa: E402

V, T = 9487, 16


def split(rng, B, R):
    seqs, gts = np.zeros((B, T), np.int64), []
    for i in range(B):
        pool = rng.randint(1, V + 1, size=20)
        ln = rng.randint(8, T + 1)
        seqs[i, :ln] = pool[rng.randint(0, 20, size=ln)]
        refs = np.zeros((R, T), np.int32)
        for r in range(R):
            ln = rng.randint(8, T + 1)
            refs[r, :ln] = pool[rng.randint(0, 20, size=ln)]
        gts.append(refs)
    return seqs, gts


def stats(ms):
    return {'ms': round(statistics.median(ms), 4), 'ms_min': round(min(ms), 4), 'ms_max': round(max(ms), 4)}


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--images', type=int, default=5000)
    p.add_argument('--refs', type=int, default=5)
    p.add_argument('--steps', type=int, default=5)
    p.add_argument('--windows', type=int, default=7)
    a = p.parse_args()
    from imagecaptioning.pytorch_b200 import _lib, eval_multi, rewards
    out = dict(device_info())
    seqs, gts = split(np.random.RandomState(0), a.images, a.refs)
    seq = torch.from_numpy(seqs).cuda()
    eval_multi.coco_scores(seq, gts)                                  # warm-up: module load, table reservation, staging buffers
    # the kernels alone, on references packed once
    refs, offsets, L = rewards.pack_references(gts, seq.device)
    refs, offsets = refs.clone(), offsets.clone()
    S = a.images
    buf = torch.empty(4 * S + 4 + 2 * S + 3 * S, dtype=torch.float64, device='cuda')
    ptr, lib, table = _lib.ptr(buf), _lib.load(), eval_multi._coco_table._h

    def kernels():
        _lib.check(lib.capb200_coco_scores(table, _lib.ptr(seq), S, 1, T, _lib.ptr(refs), _lib.ptr(offsets), L, ptr, ptr + 8 * 4 * S,
                                           ptr + 8 * (4 * S + 4), ptr + 8 * (5 * S + 4), ptr + 8 * (6 * S + 4), _lib.current_stream()), 'coco_scores')
    kernels()
    torch.cuda.synchronize()
    k_ms = []
    for _ in range(a.windows):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.steps):
            kernels()
        e1.record()
        e1.synchronize()
        k_ms.append(e0.elapsed_time(e1) / a.steps)
    e_ms = []
    for _ in range(a.windows):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(a.steps):
            res = eval_multi.coco_scores(seq, gts)                   # ends in a device-to-host copy: synchronised
        e_ms.append(1e3 * (time.perf_counter() - t0) / a.steps)
    out.update({'images': a.images, 'refs_per_image': a.refs, 'T': T, 'kernels': stats(k_ms), 'coco_scores': stats(e_ms),
                'overall': {k: round(v, 6) for k, v in res['overall'].items()}})
    print(json.dumps(out))


if __name__ == '__main__':
    main()
