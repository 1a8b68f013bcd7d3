"""Shared helpers for the parity tests."""
import argparse
import contextlib
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


# ---- dropout masks of the fused training steps, regenerated from the engine's Philox streams (capb200.h lists the sites) -----------------

def _mask_fn(b200, seed):
    L, lib = b200._lib, b200._lib.load()

    def mask(site, step, shape, p):
        n = int(np.prod(shape))
        m = torch.empty(n, device='cuda')
        L.check(lib.capb200_dropout_mask(L.ptr(m), n, seed, site, step, p, L.current_stream()), 'dropout_mask')
        return m.cpu().reshape(shape)
    return mask


def dropout_masks(b200, seed, p, B, R, N, T, E, H):
    """UpDown: fc_embed [B, H], att_embed [B, R, H], the word embedding [T, N, E] and the LSTM output [T, N, H]."""
    mask = _mask_fn(b200, seed)
    return {'fc': mask(0, 0, (B, H), p), 'att': mask(1, 0, (B, R, H), p),
            'xt': torch.stack([mask(2, t, (N, E), p) for t in range(T)]), 'out': torch.stack([mask(3, t, (N, H), p) for t in range(T)])}


def att2in2_masks(b200, seed, p, B, R, N, T, E, H):
    """Att2in2: att_embed [B, R, H], the word embedding [T, N, E] and the core output [T, N, H]."""
    d = dropout_masks(b200, seed, p, B, R, N, T, E, H)
    del d['fc']
    return d


def aoa_masks(b200, seed, B, R, N, T, E, H, heads, p_lm, p_at, p_aoa, p_sub):
    """Every dropout mask of one AoANet training step: att_embed, the refiner's attention / AoA / sublayer sites, then per step the word,
    ctx, decoder attention and output sites."""
    mask = _mask_fn(b200, seed)
    d = {'att': mask(1, 0, (B, R, H), p_lm)}
    for l in range(6):
        d['ref_p%d' % l] = mask(10 + l, 0, (B, heads, R, R), p_at)
        d['ref_aoa%d' % l] = mask(20 + l, 0, (B, R, 2 * H), p_aoa)
        d['ref_sub%d' % l] = mask(30 + l, 0, (B, R, H), p_sub)
    d['xt'] = torch.stack([mask(2, t, (N, E), p_lm) for t in range(T)])
    d['out'] = torch.stack([mask(3, t, (N, H), p_lm) for t in range(T)])
    d['ctx'] = torch.stack([mask(4, t, (N, H), p_lm) for t in range(T)])
    d['p'] = torch.stack([mask(5, t, (N, heads, 1, R), p_at) for t in range(T)])
    return d


def tfm_masks(b200, seed, B, R, N, L, T, D, Dff, heads, layers, p_lm, p):
    """Every dropout mask of one Transformer training step over L decoder positions (T = the model's seq_length): att_embed, per encoder
    layer the attention / sublayer / feed-forward sites, the positional embedding and per decoder layer its sites, one stream per
    position (element index n * cols + c)."""
    mask = _mask_fn(b200, seed)

    def per_t(site, shape):            # decoder tensors  ->  [N, L, ...]
        return torch.stack([mask(site, t, shape, p) for t in range(L)], 1)
    idxL = T + 2
    d = {'att_embed': mask(1, 0, (B, R, D), p_lm), 'emb': per_t(2, (N, D))}
    for l in range(layers):
        d['enc_p%d' % l] = mask(10 + l, 0, (B, heads, R, R), p)
        d['enc_sub0_%d' % l] = mask(20 + l, 0, (B, R, D), p)
        d['enc_ffn%d' % l] = mask(30 + l, 0, (B, R, Dff), p)
        d['enc_sub1_%d' % l] = mask(40 + l, 0, (B, R, D), p)
        d['dec_p%d' % l] = mask(50 + l, 0, (N, heads, idxL, idxL), p)[:, :, :L, :L]
        d['dec_sub0_%d' % l] = per_t(60 + l, (N, D))
        d['dec_src%d' % l] = per_t(70 + l, (N, heads, R)).permute(0, 2, 1, 3)          # [N, L, heads, R] -> [N, heads, L, R]
        d['dec_sub1_%d' % l] = per_t(80 + l, (N, D))
        d['dec_ffn%d' % l] = per_t(90 + l, (N, Dff))
        d['dec_sub2_%d' % l] = per_t(100 + l, (N, D))
    return d


# ---- Transformer ReLUs: feed-forward pre-activations, and biases that keep them clear of the kink ------------------------------------

@contextlib.contextmanager
def ffn_relu_inputs(on_input):
    """Runs the oracle's feed-forward layers (caption_oracle._ffn) through ``on_input(prefix, W, a)``, called with each layer's w_1
    pre-activations ``a`` before the ReLU, in the order the layers run; it returns the pre-activations the layer goes on with (and may
    change W[prefix + 'w_1.bias'] to match).  The layer's GEMMs resolve co.linear at call time, as the oracle's own do."""
    orig = co._ffn

    def ffn(W, pre, x, h_drop=None):
        hdn = torch.relu(on_input(pre, W, co.linear(x, W[pre + 'w_1.weight'], W[pre + 'w_1.bias'])))
        if h_drop is not None:
            hdn = hdn * h_drop
        return co.linear(hdn, W[pre + 'w_2.weight'], W[pre + 'w_2.bias'])
    co._ffn = ffn
    try:
        yield
    finally:
        co._ffn = orig


def _clear_units(a, b, margin, max_steps):
    """New fp32 bias b' (float64 [H]) for the pre-activations a [rows, H] (computed with bias b) such that every |a - b + b'| is at least
    margin x RMS(a): each unit with a row inside the band moves by the smallest +-k x margin x RMS (k = 1, 2, ...; + before -) that
    clears all its rows, rounded to fp32 as the engine holds it.  Returns (b', RMS)."""
    rms = float(a.pow(2).mean().sqrt())
    band = margin * rms
    amb = (a.abs() < band).any(0).nonzero().flatten()
    b_new = b.clone()
    if len(amb):
        z = a[:, amb] - b[amb]                                 # the bias-free part of each ambiguous unit
        todo = torch.ones(len(amb), dtype=torch.bool)
        for k in range(1, max_steps + 1):
            for sign in (1.0, -1.0):
                cand = (b[amb] + sign * k * band).float().double()
                # 0.1 % over the band: the RMS moves slightly once the units are shifted, and the check that follows recomputes it
                ok = todo & ((z + cand).abs() >= 1.001 * band).all(0)
                b_new[amb[ok]] = cand[ok]
                todo &= ~ok
            if not bool(todo.any()):
                break
        assert not bool(todo.any()), ('units with no clearing shift within %d margins' % max_steps, amb[todo].tolist())
    return b_new, rms


def clear_relu_kinks(W, att, forward, margin, max_steps=200):
    """The Transformer's weights with every ReLU decisive: W {name: fp32 tensor} with att_embed's and each feed-forward w_1's bias shifted
    so that no float64 pre-activation of the step lies within ``margin`` x the layer's RMS of zero.  A unit within rounding of its kink can
    be on in one fp32 implementation and off in another, and its flip moves the gradient of every tensor upstream of it; moving the model
    off the kinks lets every gradient tensor be compared in full.

    ``att`` holds the region features (every region counts, masked or not); ``forward(W64)`` runs the step's float64 forward through the
    oracle (its tokens, region masks and replayed dropout masks), which calls the encoder's and then the decoder's feed-forward layers in
    order, so each layer is cleared on the inputs the already-shifted earlier layers give it.  Every row counts, including rows whose
    gradient is zero (padding, finished samples, masked regions).  Returns (shifted fp32 weights, {layer: units shifted}, largest shift
    as a fraction of its layer's RMS)."""
    W64 = {k: v.detach().double().clone() for k, v in W.items()}
    shifted, largest = {}, [0.0]

    def clear(name, a, b):
        b_new, rms = _clear_units(a, b, margin, max_steps)
        moved = b_new != b
        shifted[name] = int(moved.sum())
        largest[0] = max(largest[0], float((b_new - b).abs().max()) / rms)
        return b_new

    x = att.double().reshape(-1, att.shape[-1])
    b = W64['att_embed.0.bias']
    W64['att_embed.0.bias'] = clear('att_embed', co.linear(x, W64['att_embed.0.weight'], b), b)

    def on_input(pre, Wd, a):
        b = Wd[pre + 'w_1.bias']
        b_new = clear(pre[len('model.'):-len('.feed_forward.')], a.reshape(-1, a.shape[-1]), b)
        Wd[pre + 'w_1.bias'] = b_new
        return a + (b_new - b)
    with torch.no_grad(), ffn_relu_inputs(on_input):
        forward(W64)
    out = {k: v.clone() for k, v in W.items()}
    for k in out:
        if k == 'att_embed.0.bias' or k.endswith('w_1.bias'):
            out[k] = W64[k].float()
    return out, shifted, largest[0]


def relu_inputs(W, att, forward, linear=None):
    """[(layer, pre-activations [rows, H])] of the Transformer's ReLUs (att_embed, then every feed-forward layer in order) for the step
    ``forward(W)`` runs, in W's dtype; ``linear`` (default co.linear) computes att_embed's."""
    out = [('att_embed', (linear or co.linear)(att.to(W['att_embed.0.weight']).reshape(-1, att.shape[-1]), W['att_embed.0.weight'],
                                               W['att_embed.0.bias']).detach())]

    def on_input(pre, Wd, a):
        out.append((pre[len('model.'):-len('.feed_forward.')], a.detach().reshape(-1, a.shape[-1])))
        return a
    with torch.no_grad(), ffn_relu_inputs(on_input):
        forward(W)
    return out


# ---- gradients against a float64 reference, with a bar calibrated by the fp32 oracle's own distance from it ------------------------------

def grad_bar(err32, ref_scale, largest, floor=2e-6, factor=4.0):
    """max(factor x the calibrating oracle's error, floor x the float64 tensor's size) + 1e-7 x the step's largest gradient entry."""
    return max(factor * err32, floor * ref_scale) + 1e-7 * largest


def check_grads_f64(named, ref64, ref32, keep=None, zero_rel=1e-12, label='', floor=2e-6, factor=4.0):
    """Every engine gradient (``named``: {name: tensor}) against float64 autograd ``ref64``, in max-abs and in Frobenius norm, each held to
    grad_bar with the oracle ``ref32`` supplying the error an implementation of the same arithmetic makes (fp32, or the engine mode's).  ``keep`` {name: bool mask} leaves out
    the entries float64 cannot decide (gradients routed through a ReLU whose input is within rounding of zero).  A tensor whose float64
    gradient is zero (softmax shift invariance: alpha_net.bias, attention key biases) holds rounding noise only and is held to 4x the fp32
    oracle's noise or 1e-6 of the step's largest gradient.  Prints, per tensor, the error as a fraction of its bar and the oracle's own
    error relative to the tensor; returns the worst fraction."""
    assert set(named) == set(ref64), set(named) ^ set(ref64)
    largest = max(float(v.abs().max()) for v in ref64.values())
    failures, worst = [], (0.0, '')
    for k in sorted(named):
        g, r64, r32 = named[k].detach().cpu().double(), ref64[k], ref32[k].double()
        if keep is not None and k in keep:
            g, r64, r32 = g[keep[k]], r64[keep[k]], r32[keep[k]]
        scale = float(r64.abs().max())
        e, e32 = (g - r64).abs(), (r32 - r64).abs()
        if scale <= zero_rel * largest:
            bar = max(factor * float(e32.max()), 1e-6 * largest)
            ratio = float(e.max()) / bar
            rel32 = float(e32.max()) / largest
        else:
            bar = grad_bar(float(e32.max()), scale, largest, floor, factor)
            nbar = grad_bar(float(e32.norm()), float(r64.norm()), largest * e.numel() ** 0.5, floor, factor)
            ratio = max(float(e.max()) / bar, float(e.norm()) / nbar)
            rel32 = float(e32.max()) / scale
        print('%s %-45s err/bar %.3f  oracle %.2e' % (label, k, ratio, rel32))
        worst = max(worst, (ratio, k))
        if ratio > 1.0:
            failures.append((k, ratio, float(e.max()), scale))
    print('%s worst gradient err/bar %.3f (%s)' % (label, worst[0], worst[1]))
    assert not failures, failures
    # the comparison is not vacuous (NewFC has 9 tensors in all: every one of them)
    assert sum(float(v.abs().max()) > 1e-5 for v in ref64.values()) >= min(15, len(ref64))
    return worst[0]
