"""Shared helpers for the parity tests."""
import argparse
import os
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)

from oracle import caption_oracle as co   # noqa: E402  (tests are allowed to use the oracle as the checker)

LOGP_TOL = 1e-4      # BASELINE.json north_star: log-probs within 1e-4 (fp32)
PARITY_MODES = ['simt_fp32', 'tc_f16x3']


from imagecaptioning.pytorch_b200 import synthetic as syn   # noqa: E402


def family_opt(family, V, E, H, A, F_fc, F_att, T, heads=8):
    """opt namespace for a family; for 'transformer' E = d_model, H = d_ff, A = layers per stack (make_weights convention)."""
    return syn.model_opt(family, V, E, H, A, F_fc, F_att, T, heads)


def make_opt(family, V, E, H, A, F_fc, F_att, T):
    return syn.model_opt(family, V, E, H, A, F_fc, F_att, T)


def build_pair(family, V, E, H, A, F_fc, F_att, T, seed, logit_scale, mode, device='cuda', heads=8):
    """Returns (engine model on the GPU, oracle Family on the CPU) sharing the same synthetic weights.
    For 'transformer': E = d_model, H = d_ff, A = layers per stack (the make_weights convention)."""
    import imagecaptioning.pytorch_b200 as b200
    W = co.make_weights(family, V, E, H, A, F_fc, F_att, seed=seed, logit_scale=logit_scale)
    model = b200.setup(family_opt(family, V, E, H, A, F_fc, F_att, T, heads), numeric_mode=mode)
    model.load_state_dict(W, strict=True)
    model = model.to(device).eval()
    return model, co.Family(family, W, T, heads=heads)


def first_divergence(a, b):
    """Index of the first column where two id matrices differ, per row (-1 = identical)."""
    a, b = np.asarray(a), np.asarray(b)
    out = np.full(a.shape[0], -1)
    for i in range(a.shape[0]):
        d = np.nonzero(a[i] != b[i])[0]
        if d.size:
            out[i] = d[0]
    return out


def check_decode(fam, fc, att, seq, lp, oseq, olp, margins, masks=None, sample_n=1, done_p=None, odone=None):
    """Non-vacuous decode comparison.
    * decisions separated by more than 10x the log-prob tolerance -> token ids must be bit-exact and log-probs within 1e-4;
    * always: the returned sequences, re-scored by the oracle with teacher forcing, must carry the log-probs the engine reported
      (within 1e-4), and for beam search the winning score must match the oracle's best score within 1e-3 -- so a legitimately
      ambiguous near-tie can change which hypothesis wins, but never produce a worse or mis-scored one."""
    import torch
    seq_c, lp_c = seq.cpu(), lp.cpu()
    strict = min(margins) > 10 * LOGP_TOL
    if strict:
        assert np.array_equal(seq_c.numpy(), oseq.numpy()), (min(margins), first_divergence(seq_c.numpy(), oseq.numpy()))
        picked = lp_c.gather(2, seq_c.unsqueeze(2)).squeeze(2)
        opicked = olp.gather(2, oseq.unsqueeze(2)).squeeze(2)
        assert float((picked - opicked).abs().max()) < LOGP_TOL
        assert bool(((lp_c - olp).abs() <= LOGP_TOL + 1e-5 * olp.abs()).all())
    N, T = seq_c.shape
    labels = torch.cat([torch.zeros(N, 1, dtype=torch.long), seq_c[:, :-1]], 1)
    B = fc.shape[0]
    tf = co.forward_teacher(fam, fc, att, labels.reshape(B, N // B, T), masks)
    valid = torch.cat([torch.ones(N, 1, dtype=torch.bool), (seq_c[:, :-1] > 0)], 1)       # tokens through the first EOS
    mine = lp_c.gather(2, seq_c.unsqueeze(2)).squeeze(2)
    theirs = tf.gather(2, seq_c.unsqueeze(2)).squeeze(2)
    assert float(((mine - theirs).abs() * valid).max()) < 2 * LOGP_TOL, float(((mine - theirs).abs() * valid).max())
    if done_p is not None and odone is not None:
        best = np.array([d[0]['p'] for d in odone])
        assert np.abs(np.asarray(done_p)[:, 0] - best).max() < 1e-3
    return strict
