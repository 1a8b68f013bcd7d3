"""Seeded synthetic data for benchmarks, smoke runs and tests: reference-shaped weights (state_dict names of the reference models),
bottom-up-style features, reference captions and a document-frequency table in the scripts/prepro_ngrams.py format.

None of this is on the product path: there is no network for checkpoints or datasets, so BASELINE.json's configurations are measured
on random-init weights of the right architecture and random features of the right shape (bench.py states ``data: synthetic``).
"""
from __future__ import annotations

import math
from collections import defaultdict
from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch

Weights = Dict[str, torch.Tensor]


def _uniform(gen, shape, bound):
    return (torch.rand(shape, generator=gen) * 2 - 1) * bound


def make_weights(family: str, V: int, E: int, H: int, A: int, F_fc: int, F_att: int, seed: int = 1234,
                 logit_scale: float = 12.0, logit_layers: int = 1) -> Weights:
    """Deterministic synthetic weights with torch-default-like ranges; ``logit.weight`` is scaled so the
    next-word distribution is peaked (top-1/top-2 margins far above the 1e-4 log-prob tolerance).  ``logit_layers`` > 1 adds the
    output head of AttModel (add_logit_head); every other tensor is drawn as with the default."""
    g = torch.Generator().manual_seed(seed)
    V1 = V + 1
    W: Weights = {}

    def lin(name, out_f, in_f, scale=1.0):
        b = 1.0 / math.sqrt(in_f)
        W[name + '.weight'] = _uniform(g, (out_f, in_f), b) * scale
        W[name + '.bias'] = _uniform(g, (out_f,), b)

    if family == 'updown':
        W['embed.0.weight'] = torch.randn(V1, E, generator=g)
        lin('fc_embed.0', H, F_fc)
        lin('att_embed.0', H, F_att)
        lin('logit', V1, H, logit_scale)
        lin('ctx2att', A, H)
        b = 1.0 / math.sqrt(H)
        for cell, in_f in (('core.att_lstm', E + 2 * H), ('core.lang_lstm', 2 * H)):
            W[cell + '.weight_ih'] = _uniform(g, (4 * H, in_f), b)
            W[cell + '.weight_hh'] = _uniform(g, (4 * H, H), b)
            W[cell + '.bias_ih'] = _uniform(g, (4 * H,), b)
            W[cell + '.bias_hh'] = _uniform(g, (4 * H,), b)
        lin('core.attention.h2att', A, H)
        lin('core.attention.alpha_net', 1, A)
    elif family == 'aoa':
        W['embed.0.weight'] = torch.randn(V1, E, generator=g)
        lin('att_embed.0', H, F_att)
        lin('logit', V1, H, logit_scale)
        lin('ctx2att', 2 * H, H)
        for i in range(6):
            pre = 'refiner.layers.%d.' % i
            for j in range(3):
                lin(pre + 'self_attn.linears.%d' % j, H, H)
            lin(pre + 'self_attn.aoa_layer.0', 2 * H, 2 * H)
            W[pre + 'sublayer.0.norm.a_2'] = 1 + 0.1 * torch.randn(H, generator=g)
            W[pre + 'sublayer.0.norm.b_2'] = 0.1 * torch.randn(H, generator=g)
        W['refiner.norm.a_2'] = 1 + 0.1 * torch.randn(H, generator=g)
        W['refiner.norm.b_2'] = 0.1 * torch.randn(H, generator=g)
        b = 1.0 / math.sqrt(H)
        W['core.att_lstm.weight_ih'] = _uniform(g, (4 * H, E + H), b)
        W['core.att_lstm.weight_hh'] = _uniform(g, (4 * H, H), b)
        W['core.att_lstm.bias_ih'] = _uniform(g, (4 * H,), b)
        W['core.att_lstm.bias_hh'] = _uniform(g, (4 * H,), b)
        lin('core.att2ctx.0', 2 * H, 2 * H)
        W['core.attention.norm.a_2'] = 1 + 0.1 * torch.randn(H, generator=g)
        W['core.attention.norm.b_2'] = 0.1 * torch.randn(H, generator=g)
        lin('core.attention.linears.0', H, H)
        W['logit.bias'][0] -= 4.0          # keep EOS from winning at the first steps so the synthetic captions have some length
    elif family == 'transformer':
        # here E = d_model, H = d_ff, A = number of layers (both stacks)
        D, Dff, NL = E, H, A

        def xav(name, out_f, in_f, scale=1.0):
            bnd = math.sqrt(6.0 / (in_f + out_f))
            W[name + '.weight'] = _uniform(g, (out_f, in_f), bnd) * scale
            W[name + '.bias'] = _uniform(g, (out_f,), 1.0 / math.sqrt(in_f))

        def norm(name):
            W[name + '.a_2'] = 1 + 0.1 * torch.randn(D, generator=g)
            W[name + '.b_2'] = 0.1 * torch.randn(D, generator=g)

        xav('att_embed.0', D, F_att)
        for stack, n_sub in (('encoder', 2), ('decoder', 3)):
            for i in range(NL):
                pre = 'model.%s.layers.%d.' % (stack, i)
                for att_name in (('self_attn',) if stack == 'encoder' else ('self_attn', 'src_attn')):
                    for j in range(4):
                        xav(pre + att_name + '.linears.%d' % j, D, D)
                xav(pre + 'feed_forward.w_1', Dff, D)
                xav(pre + 'feed_forward.w_2', D, Dff)
                for j in range(n_sub):
                    norm(pre + 'sublayer.%d.norm' % j)
            norm('model.%s.norm' % stack)
        W['model.tgt_embed.0.lut.weight'] = torch.randn(V1, D, generator=g) * (1.0 / math.sqrt(D))
        pe = torch.zeros(5000, D)
        position = torch.arange(0, 5000).unsqueeze(1).float()
        div_term = torch.exp(torch.arange(0, D, 2).float() * -(math.log(10000.0) / D))
        pe[:, 0::2] = torch.sin(position * div_term)
        pe[:, 1::2] = torch.cos(position * div_term)
        W['model.tgt_embed.1.pe'] = pe.unsqueeze(0)
        xav('model.generator.proj', V1, D, logit_scale)
    elif family == 'att2in2':
        W['embed.0.weight'] = torch.randn(V1, E, generator=g)
        lin('att_embed.0', H, F_att)
        lin('logit', V1, H, logit_scale)
        lin('ctx2att', A, H)
        lin('core.a2c', 2 * H, H)
        lin('core.i2h', 5 * H, E)
        lin('core.h2h', 5 * H, H)
        lin('core.attention.h2att', A, H)
        lin('core.attention.alpha_net', 1, A)
    elif family == 'newfc':
        W['embed.weight'] = torch.randn(V1, E, generator=g)
        lin('fc_embed', E, F_fc)
        lin('logit', V1, H, logit_scale)
        lin('_core.i2h', 5 * H, E)
        lin('_core.h2h', 5 * H, H)
    else:
        raise ValueError(family)
    if logit_layers > 1 and family != 'transformer':      # the Transformer has no self.logit (TransformerModel.py:285)
        add_logit_head(W, H, logit_layers, seed)
    return W


def add_logit_head(W: Weights, H: int, logit_layers: int, seed: int) -> Weights:
    """Turns W's vocabulary Linear into AttModel's head for logit_layers = k > 1 (AttModel.py:87-92): k - 1 hidden Linear(H, H) layers
    logit.0, logit.3, ... (each followed by ReLU and Dropout in the reference) ahead of the vocabulary Linear, renamed logit.{3(k-1)}.
    The hidden layers come from a generator of their own, with a gain of sqrt(6) that keeps the ReLU outputs at the scale of their
    inputs, so the vocabulary rows stay as peaked as without a head."""
    g = torch.Generator().manual_seed(seed + 7919)
    b = 1.0 / math.sqrt(H)
    for i in range(logit_layers - 1):
        W['logit.%d.weight' % (3 * i)] = _uniform(g, (H, H), b) * math.sqrt(6.0)
        W['logit.%d.bias' % (3 * i)] = _uniform(g, (H,), b)
    last = 3 * (logit_layers - 1)
    W['logit.%d.weight' % last] = W.pop('logit.weight')
    W['logit.%d.bias' % last] = W.pop('logit.bias')
    return W


def make_inputs(B: int, R: int, F_fc: int, F_att: int, seed: int = 1234):
    g = torch.Generator().manual_seed(seed + 1)
    return torch.randn(B, F_fc, generator=g), torch.randn(B, R, F_att, generator=g)


def make_refs(B: int, V: int, n_refs: int = 5, L: int = 16, seed: int = 7, zipf: bool = True) -> List[np.ndarray]:
    """Synthetic references: per image n_refs rows, lengths U[6,15], 0-padded to L.  Ids follow a Zipf-like law so
    n-grams repeat (otherwise every similarity would be 0)."""
    rng = np.random.RandomState(seed)
    out = []
    for _ in range(B):
        rows = np.zeros((n_refs, L), dtype=np.int64)
        for j in range(n_refs):
            ln = rng.randint(6, 16)
            if zipf:
                ids = np.minimum(rng.zipf(1.3, size=ln), V).astype(np.int64)
            else:
                ids = rng.randint(1, V + 1, size=ln)
            rows[j, :ln] = ids
        out.append(rows)
    return out


def document_frequency(ref_rows_per_image: Sequence[Sequence[Sequence[int]]], max_n: int = 4):
    """Data preparation in the format of scripts/prepro_ngrams.py (:26, :42-45): for every n-gram (n <= 4) of the reference rows, cut
    through the first 0 (<eos>), the number of images whose references contain it.  Returns (table, number of images = ref_len)."""
    df: Dict[Tuple[int, ...], float] = defaultdict(float)
    for rows in ref_rows_per_image:
        seen = set()
        for row in rows:
            toks = []
            for t in row:
                toks.append(int(t))
                if int(t) == 0:
                    break
            for n in range(1, max_n + 1):
                for i in range(len(toks) - n + 1):
                    seen.add(tuple(toks[i:i + n]))
        for gram in seen:
            df[gram] += 1.0
    return dict(df), len(ref_rows_per_image)


def model_opt(family: str, V: int, E: int, H: int, A: int, F_fc: int, F_att: int, T: int, heads: int = 8, logit_layers: int = 1):
    """argparse-style ``opt`` of the reference for one family (for 'transformer': E = d_model, H = d_ff, A = layers per stack)."""
    import argparse
    opt = argparse.Namespace(vocab_size=V, input_encoding_size=E, rnn_size=H, num_layers=1, drop_prob_lm=0.5, max_length=T, seq_length=T,
                             fc_feat_size=F_fc, att_feat_size=F_att, att_hid_size=A, vocab={str(i): 'w%d' % i for i in range(1, V + 1)},
                             caption_model=family, use_bn=0, logit_layers=logit_layers)
    if family == 'transformer':
        opt.num_layers, opt.N_enc, opt.N_dec, opt.d_model, opt.d_ff, opt.num_att_heads = A, A, A, E, H, heads
    if family == 'aoa':
        opt.num_layers, opt.refine, opt.refine_aoa, opt.use_ff, opt.decoder_type, opt.use_multi_head = 2, 1, 1, 0, 'AoA', 2
        opt.num_heads, opt.multi_head_scale, opt.mean_feats, opt.ctx_drop = heads, 1, 1, 1
    return opt


def build_model(family: str, V: int, E: int, H: int, A: int, F_fc: int, F_att: int, T: int, seed: int, logit_scale: float, mode: str,
                device='cuda', heads: int = 8, logit_layers: int = 1):
    """Engine model of ``family`` with the seeded synthetic weights loaded, on ``device``, in eval mode."""
    from . import setup
    W = make_weights(family, V, E, H, A, F_fc, F_att, seed=seed, logit_scale=logit_scale, logit_layers=logit_layers)
    model = setup(model_opt(family, V, E, H, A, F_fc, F_att, T, heads, logit_layers), numeric_mode=mode)
    model.load_state_dict(W, strict=True)
    return model.to(device).eval()
