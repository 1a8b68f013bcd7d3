"""Time of the caption-set diversity scores: the device path against the reference's CPU functions.

    python tools/diversity_rate.py [--images 5000] [--ns 5 10] [--steps 5] [--windows 5] [--ref-images 5000]

For each n, --images images x n captions (T = 16, V = 9487, seeded ids from a per-image pool of words, so captions share n-grams):
* device: rewards.get_self_cider_scores (the self-CIDEr matrices + eigenvalue diversity, with a pickle-style table) and
  eval_multi.div_stats (Div-1, Div-2, gDiv-1, mutual BLEU, one host transfer included), ms per call as the median over --windows windows
  of --steps calls;
* reference: the unmodified rewards.get_self_cider_scores after init_scorer reads the same df pickle, and eval_div_stats' statistics
  (div_utils.compute_div_n / compute_global_div_n and the n Bleu(4) leave-one-out rounds on 'w<id>' words, without the Java tokenizer),
  one timed call each over --ref-images images, from oracle/_ref/ when that copy is present.
Prints one JSON line with the device name and power limit of the same run.
"""
from __future__ import annotations

import argparse
import collections
import contextlib
import io
import json
import os
import pickle
import shutil
import sys
import tempfile
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tools'))

from dbs_rate import device_info                  # noqa: E402
from reward_rate import summary, windows          # noqa: E402

V, T = 9487, 16


def caption_sets(rng, B, n):
    seqs = np.zeros((B * n, T), np.int64)
    for i in range(B):
        pool = rng.randint(1, V + 1, size=20)
        for j in range(n):
            ln = rng.randint(6, T)
            seqs[i * n + j, :ln] = pool[rng.randint(0, 20, size=ln)]
    return seqs


def reference_times(seqs, n, df, ref_len):
    """One timed call of each reference function over `seqs`: the unmodified modules of the oracle/_ref copy, imported from a scratch
    directory that holds the cwd-relative names they expect (cider, coco-caption, data/<df>.p; captioning/utils/rewards.py:12,15)."""
    ref = os.path.join(REPO, 'oracle', '_ref')
    scratch = tempfile.mkdtemp(prefix='refcwd_')
    try:
        for name in ('cider', 'coco-caption'):
            os.symlink(os.path.join(ref, name), os.path.join(scratch, name))
        os.makedirs(os.path.join(scratch, 'data'))
        dd = collections.defaultdict(float)
        dd.update({tuple(str(t) for t in k): float(v) for k, v in df.items()})
        with open(os.path.join(scratch, 'data', 'diversity-df.p'), 'wb') as f:
            pickle.dump({'document_frequency': dd, 'ref_len': ref_len}, f, protocol=2)
        os.chdir(scratch)
        sys.path.insert(0, ref)
        with contextlib.redirect_stdout(io.StringIO()):                   # the reference prints every score
            from captioning.utils import rewards as R
            from captioning.utils import div_utils
            from pycocoevalcap.bleu.bleu import Bleu
            R.init_scorer('diversity-df')
            B = seqs.shape[0] // n
            t0 = time.perf_counter()
            R.get_self_cider_scores([None] * B, torch.from_numpy(seqs), argparse.Namespace())
            t_self = time.perf_counter() - t0
            caps = {i: [' '.join('w%d' % v for v in r[:np.argmin(r != 0) if (r == 0).any() else T]) for r in seqs[i * n:(i + 1) * n]]
                    for i in range(B)}
            t0 = time.perf_counter()
            div_utils.compute_div_n(caps, 1)
            div_utils.compute_div_n(caps, 2)
            div_utils.compute_global_div_n(caps, 1)
            bleu = Bleu(4)
            for j in range(n):
                bleu.compute_score({k: caps[k][:j] + caps[k][j + 1:] for k in caps}, {k: [caps[k][j]] for k in caps})
            t_div = time.perf_counter() - t0
    finally:
        os.chdir(REPO)
        shutil.rmtree(scratch, ignore_errors=True)
    return 1e3 * t_self, 1e3 * t_div


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--images', type=int, default=5000)
    p.add_argument('--ns', type=int, nargs='+', default=[5, 10])
    p.add_argument('--steps', type=int, default=5)
    p.add_argument('--windows', type=int, default=5)
    p.add_argument('--ref-images', type=int, default=5000)
    a = p.parse_args()
    import imagecaptioning.pytorch_b200 as b200
    out = dict(device_info())
    rng = np.random.RandomState(0)
    for n in a.ns:
        seqs = caption_sets(rng, a.images, n)
        df, ref_len = b200.eval_multi.document_frequency([seqs[i * n:i * n + 5] for i in range(a.images)])
        b200.rewards.reset_scorer()
        b200.rewards.init_scorer(b200.rewards.CiderDTable(df, ref_len))
        d = torch.from_numpy(seqs).cuda()
        gts = [None] * a.images
        b200.rewards.get_self_cider_scores(gts, d, None)
        b200.eval_multi.div_stats(d, n, vocab_size=V)
        res = {'self_cider': summary(windows(lambda i: b200.rewards.get_self_cider_scores(gts, d, None), a.steps, a.windows)),
               'div_stats': summary(windows(lambda i: b200.eval_multi.div_stats(d, n, vocab_size=V), a.steps, a.windows, sync=False))}
        b200.rewards.reset_scorer()
        if os.path.isdir(os.path.join(REPO, 'oracle', '_ref', 'captioning')) and a.ref_images > 0:
            k = min(a.ref_images, a.images)
            t_self, t_div = reference_times(seqs[:k * n], n, df, ref_len)
            res['reference_cpu'] = {'images': k, 'self_cider_ms': round(t_self, 1), 'div_stats_ms': round(t_div, 1)}
            scale = a.images / k
            res['speedup'] = {'self_cider': round(t_self * scale / res['self_cider']['ms'], 1), 'div_stats': round(t_div * scale / res['div_stats']['ms'], 1)}
        out['n%d' % n] = dict(images=a.images, **res)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
