"""CPU oracle for the caption-decode hot path (TEST INFRASTRUCTURE ONLY).

This file is a from-scratch, functional restatement (torch on CPU, no nn.Module; fp32, or float64 when given float64 weights and features) of the
reference algorithm on the path BASELINE.json names.  It is the *checker*: only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline / ``--impl reference`` leg may import it.
The product package (``imagecaptioning.pytorch_b200``) never does.

Parity pin: ``oracle/make_golden.py`` imports the live reference from ``/root/reference`` (in the build
container only) and writes ``tests/golden/*.npz``; ``tests/test_oracle_golden.py`` checks every function
here against those vectors, so this restatement is pinned to outputs of the reference itself.

Reference lines each function follows (paths relative to /root/reference/captioning):
  linear / lstm_cell        torch.nn.Linear / torch.nn.LSTMCell call sites models/AttModel.py:620-621
  updown_prepare            models/AttModel.py:114-124  (_prepare_feature; fc_embed/att_embed/ctx2att :74-95)
  additive_attention        models/AttModel.py:728-748  (Attention.forward)
  updown_core               models/AttModel.py:624-640  (UpDownCore.forward)
  newfc_prepare/newfc_core  models/AttModel.py:915-945, models/FCModel.py:25-42 (maxout LSTMCore)
  logprobs_state            models/AttModel.py:166-176  (get_logprobs_state)
  beam_search               models/CaptionModel.py:35-209 (group_size == 1 path)
  sample_beam               models/AttModel.py:218-256
  sample                    models/AttModel.py:258-352 + models/CaptionModel.py:370-407 (greedy / multinomial)
  forward_teacher           models/AttModel.py:126-164
  reward_criterion          modules/losses.py:22-37

Weights are passed as a plain dict keyed by the reference ``state_dict`` names (SURVEY.md section 8b).
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

Tensor = torch.Tensor
Weights = Dict[str, Tensor]


# --------------------------------------------------------------------------------------------------
# primitive ops
# --------------------------------------------------------------------------------------------------

def linear(x: Tensor, w: Tensor, b: Optional[Tensor] = None) -> Tensor:
    y = x @ w.t()
    return y if b is None else y + b


def lstm_cell(x: Tensor, h: Tensor, c: Tensor, w_ih: Tensor, w_hh: Tensor, b_ih: Tensor, b_hh: Tensor):
    """nn.LSTMCell arithmetic, gate order (i, f, g, o)."""
    gates = linear(x, w_ih, b_ih) + linear(h, w_hh, b_hh)
    hs = h.shape[1]
    gi, gf, gg, go = gates[:, :hs], gates[:, hs:2 * hs], gates[:, 2 * hs:3 * hs], gates[:, 3 * hs:]
    c_new = torch.sigmoid(gf) * c + torch.sigmoid(gi) * torch.tanh(gg)
    h_new = torch.sigmoid(go) * torch.tanh(c_new)
    return h_new, c_new


def repeat_rows(x: Optional[Tensor], n: int) -> Optional[Tensor]:
    """Row i*n+j of the result is row i of x (models/utils.py:3-15)."""
    if x is None or n == 1:
        return x
    return x.unsqueeze(1).expand(x.shape[0], n, *x.shape[1:]).reshape(x.shape[0] * n, *x.shape[1:])


# --------------------------------------------------------------------------------------------------
# UpDown (TopDown attention LSTM)
# --------------------------------------------------------------------------------------------------

def clip_att(att: Tensor, masks: Optional[Tensor]):
    if masks is None:
        return att, None
    max_len = int(masks.long().sum(1).max())
    return att[:, :max_len].contiguous(), masks[:, :max_len].contiguous()


def updown_prepare(W: Weights, fc: Tensor, att: Tensor, masks: Optional[Tensor] = None, drop=None):
    """fc_embed, att_embed (Linear+ReLU; dropout is identity in eval) and ctx2att.  ``drop`` (train mode) carries explicit inverted-
    dropout masks {'fc': [B,H], 'att': [B,R,H], 'xt': [T,N,E], 'out': [T,N,H]} so a run can be replayed exactly."""
    att, masks = clip_att(att, masks)
    fc_e = torch.relu(linear(fc, W['fc_embed.0.weight'], W['fc_embed.0.bias']))
    att_e = torch.relu(linear(att, W['att_embed.0.weight'], W['att_embed.0.bias']))
    if drop is not None:
        fc_e = fc_e * drop['fc']
        att_e = att_e * drop['att']
    if masks is not None:
        # pack_wrapper runs the module on valid rows only and zero-pads the rest
        att_e = att_e * masks.unsqueeze(-1).to(att_e)
    p_att = linear(att_e, W['ctx2att.weight'], W['ctx2att.bias'])
    return fc_e, att_e, p_att, masks


def additive_attention(W: Weights, h: Tensor, att_e: Tensor, p_att: Tensor, masks: Optional[Tensor], prefix='core.attention.'):
    att_h = linear(h, W[prefix + 'h2att.weight'], W[prefix + 'h2att.bias'])          # [N, A]
    dot = torch.tanh(p_att + att_h.unsqueeze(1))                                     # [N, R, A]
    score = linear(dot, W[prefix + 'alpha_net.weight'], W[prefix + 'alpha_net.bias']).squeeze(-1)   # [N, R]
    weight = F.softmax(score, dim=1)
    if masks is not None:
        weight = weight * masks.to(weight)
        weight = weight / weight.sum(1, keepdim=True)
    return torch.bmm(weight.unsqueeze(1), att_e).squeeze(1)


def updown_core(W: Weights, xt: Tensor, fc_e: Tensor, att_e: Tensor, p_att: Tensor, state, masks=None, out_drop=None):
    h, c = state                                   # each [2, N, H]
    x1 = torch.cat([h[1], fc_e, xt], 1)
    h_att, c_att = lstm_cell(x1, h[0], c[0], W['core.att_lstm.weight_ih'], W['core.att_lstm.weight_hh'],
                             W['core.att_lstm.bias_ih'], W['core.att_lstm.bias_hh'])
    att = additive_attention(W, h_att, att_e, p_att, masks)
    x2 = torch.cat([att, h_att], 1)
    h_lang, c_lang = lstm_cell(x2, h[1], c[1], W['core.lang_lstm.weight_ih'], W['core.lang_lstm.weight_hh'],
                               W['core.lang_lstm.bias_ih'], W['core.lang_lstm.bias_hh'])
    out = h_lang if out_drop is None else h_lang * out_drop       # F.dropout on the output only; the state keeps h_lang (AttModel.py:637-638)
    return out, (torch.stack([h_att, h_lang]), torch.stack([c_att, c_lang]))


# --------------------------------------------------------------------------------------------------
# NewFC (maxout LSTM fed with the image embedding at the first step)
# --------------------------------------------------------------------------------------------------

def newfc_prepare(W: Weights, fc: Tensor, att: Tensor, masks=None):
    return linear(fc, W['fc_embed.weight'], W['fc_embed.bias']), att, att, masks


def maxout_lstm(W: Weights, x: Tensor, state):
    h, c = state                                   # [1, N, H]
    hs = h.shape[2]
    s = linear(x, W['_core.i2h.weight'], W['_core.i2h.bias']) + linear(h[-1], W['_core.h2h.weight'], W['_core.h2h.bias'])
    sig = torch.sigmoid(s[:, :3 * hs])
    i_g, f_g, o_g = sig[:, :hs], sig[:, hs:2 * hs], sig[:, 2 * hs:3 * hs]
    g = torch.max(s[:, 3 * hs:4 * hs], s[:, 4 * hs:5 * hs])
    c_new = f_g * c[-1] + i_g * g
    h_new = o_g * torch.tanh(c_new)
    return h_new, (h_new.unsqueeze(0), c_new.unsqueeze(0))


def newfc_core(W: Weights, xt: Tensor, fc_e: Tensor, att_e, p_att, state, masks=None):
    first = (state[0] == 0).all(2).all(0)          # rows whose state is exactly zero
    if bool(first.all()):
        _, state = maxout_lstm(W, fc_e, state)
    elif bool(first.any()):
        _, st2 = maxout_lstm(W, fc_e, state)
        state = (torch.where(first[None, :, None], st2[0], state[0]), torch.where(first[None, :, None], st2[1], state[1]))
    return maxout_lstm(W, xt, state)


# --------------------------------------------------------------------------------------------------
# Transformer (annotated-transformer encoder/decoder) and AoA (attention-on-attention) pieces
#   layer_norm          models/TransformerModel.py:76-87   (unbiased std, eps added to the std)
#   dot_attention       models/TransformerModel.py:152-162
#   mha4                models/TransformerModel.py:164-195 (four Linears: q, k, v, out)
#   transformer_encode  models/TransformerModel.py:305-338 + Encoder/EncoderLayer :64-115
#   transformer_decode  models/TransformerModel.py:351-363 (stateless: re-runs all t tokens) + Decoder/DecoderLayer :117-144
#   aoa_prepare         models/AoAModel.py:207-226 (+ AoA_Refiner_Core/Layer :100-126, MultiHeadedDotAttention :56-98)
#   aoa_core            models/AoAModel.py:163-186
# --------------------------------------------------------------------------------------------------

def layer_norm(x: Tensor, a: Tensor, b: Tensor, eps: float = 1e-6) -> Tensor:
    mean = x.mean(-1, keepdim=True)
    std = x.std(-1, keepdim=True)
    return a * (x - mean) / (std + eps) + b


def dot_attention(q: Tensor, k: Tensor, v: Tensor, mask: Optional[Tensor], p_drop: Optional[Tensor] = None) -> Tensor:
    """captioning/models/TransformerModel.py:152-162; ``p_drop`` is an explicit keep/scale mask for the dropout on the
    attention probabilities (:160-161), shaped like the probabilities [n, h, tq, tk]."""
    scores = torch.matmul(q, k.transpose(-2, -1)) / math.sqrt(q.shape[-1])
    if mask is not None:
        scores = scores.masked_fill(mask == 0, float('-inf'))
    p = F.softmax(scores, dim=-1)
    if p_drop is not None:
        p = p * p_drop
    return torch.matmul(p, v)


def _heads(x: Tensor, h: int) -> Tensor:
    n, t, d = x.shape
    return x.view(n, t, h, d // h).transpose(1, 2)


def mha4(W: Weights, pre: str, q: Tensor, k: Tensor, v: Tensor, mask: Optional[Tensor], h: int, p_drop: Optional[Tensor] = None) -> Tensor:
    if mask is not None:
        mask = mask.unsqueeze(1)
    qh, kh, vh = (_heads(linear(x, W[pre + 'linears.%d.weight' % i], W[pre + 'linears.%d.bias' % i]), h) for i, x in enumerate((q, k, v)))
    x = dot_attention(qh, kh, vh, mask, p_drop).transpose(1, 2).contiguous().view(q.shape[0], -1, q.shape[2])
    return linear(x, W[pre + 'linears.3.weight'], W[pre + 'linears.3.bias'])


def _ffn(W: Weights, pre: str, x: Tensor, h_drop: Optional[Tensor] = None) -> Tensor:
    """PositionwiseFeedForward (TransformerModel.py:197-206); ``h_drop`` = explicit keep/scale mask of the dropout between w_1 and w_2."""
    hdn = torch.relu(linear(x, W[pre + 'w_1.weight'], W[pre + 'w_1.bias']))
    if h_drop is not None:
        hdn = hdn * h_drop
    return linear(hdn, W[pre + 'w_2.weight'], W[pre + 'w_2.bias'])


def _dm(drop, key, x: Tensor) -> Tensor:
    """x * drop[key] when a train-mode replay supplies that mask (explicit keep/scale masks stand in for nn.Dropout)."""
    return x if drop is None or key not in drop else x * drop[key]


def _ln(W: Weights, pre: str, x: Tensor) -> Tensor:
    return layer_norm(x, W[pre + 'a_2'], W[pre + 'b_2'])


def transformer_prepare(W: Weights, fc: Tensor, att: Tensor, masks: Optional[Tensor], n_layers: int, h: int, drop=None):
    """TransformerModel._prepare_feature (:305-338).  ``drop`` (train-mode replay): 'att_embed' [B,R,D], per encoder layer i 'enc_p%d' [B,h,R,R]
    (attention probabilities), 'enc_sub0_%d' / 'enc_sub1_%d' [B,R,D] (SublayerConnection, :89-101), 'enc_ffn%d' [B,R,d_ff]."""
    att, masks = clip_att(att, masks)
    x = _dm(drop, 'att_embed', torch.relu(linear(att, W['att_embed.0.weight'], W['att_embed.0.bias'])))
    if masks is not None:
        x = x * masks.unsqueeze(-1).to(x)
    else:
        masks = torch.ones(att.shape[:2], dtype=torch.long)
    m3 = masks.unsqueeze(-2)                                   # [B, 1, R]
    for i in range(n_layers):
        pre = 'model.encoder.layers.%d.' % i
        y = _ln(W, pre + 'sublayer.0.norm.', x)
        x = x + _dm(drop, 'enc_sub0_%d' % i, mha4(W, pre + 'self_attn.', y, y, y, m3, h, None if drop is None else drop.get('enc_p%d' % i)))
        x = x + _dm(drop, 'enc_sub1_%d' % i, _ffn(W, pre + 'feed_forward.', _ln(W, pre + 'sublayer.1.norm.', x), None if drop is None else drop.get('enc_ffn%d' % i)))
    memory = _ln(W, 'model.encoder.norm.', x)
    return fc[..., :0], att[..., :0], memory, m3


def transformer_decode(W: Weights, memory: Tensor, src_mask: Tensor, ys: Tensor, n_layers: int, h: int, tgt_mask: Optional[Tensor] = None, drop=None) -> Tensor:
    """EncoderDecoder.decode (:46-47) + Decoder / DecoderLayer (:113-144).  ``drop`` (train-mode replay): 'emb' [N,t,D] (PositionalEncoding's
    dropout), per layer i 'dec_p%d' [N,h,t,t], 'dec_src%d' [N,h,t,R], 'dec_sub0_%d' / 'dec_sub1_%d' / 'dec_sub2_%d' [N,t,D], 'dec_ffn%d' [N,t,d_ff]."""
    d = memory.shape[-1]
    t = ys.shape[1]
    x = _dm(drop, 'emb', W['model.tgt_embed.0.lut.weight'][ys] * math.sqrt(d) + W['model.tgt_embed.1.pe'][:, :t])
    if tgt_mask is None:
        tgt_mask = torch.tril(torch.ones(1, t, t, dtype=torch.bool))
    g = (lambda k: None) if drop is None else drop.get
    for i in range(n_layers):
        pre = 'model.decoder.layers.%d.' % i
        y = _ln(W, pre + 'sublayer.0.norm.', x)
        x = x + _dm(drop, 'dec_sub0_%d' % i, mha4(W, pre + 'self_attn.', y, y, y, tgt_mask, h, g('dec_p%d' % i)))
        y = _ln(W, pre + 'sublayer.1.norm.', x)
        x = x + _dm(drop, 'dec_sub1_%d' % i, mha4(W, pre + 'src_attn.', y, memory, memory, src_mask, h, g('dec_src%d' % i)))
        x = x + _dm(drop, 'dec_sub2_%d' % i, _ffn(W, pre + 'feed_forward.', _ln(W, pre + 'sublayer.2.norm.', x), g('dec_ffn%d' % i)))
    return _ln(W, 'model.decoder.norm.', x)


def aoa_mha(W: Weights, pre: str, q: Tensor, k: Tensor, v: Tensor, mask: Optional[Tensor], h: int, project_k_v: bool, norm_q: bool, do_aoa: bool,
            p_drop: Optional[Tensor] = None, aoa_drop: Optional[Tensor] = None):
    """MultiHeadedDotAttention(query, value, key) -- note the reference's argument order is (query, value, key).
    Train-mode replay: ``p_drop`` multiplies the attention probabilities (AoAModel.py:83-84 -> TransformerModel.py:160-161) and
    ``aoa_drop`` the input cat[x, query] of the AoA layer (AoAModel.py:90-92)."""
    if mask is not None:
        if mask.dim() == 2:
            mask = mask.unsqueeze(-2)
        mask = mask.unsqueeze(1)
    single = q.dim() == 2
    if single:
        q = q.unsqueeze(1)
    if norm_q:
        q = layer_norm(q, W[pre + 'norm.a_2'], W[pre + 'norm.b_2'])
    qh = _heads(linear(q, W[pre + 'linears.0.weight'], W[pre + 'linears.0.bias']), h)
    if project_k_v:
        kh = _heads(linear(k, W[pre + 'linears.1.weight'], W[pre + 'linears.1.bias']), h)
        vh = _heads(linear(v, W[pre + 'linears.2.weight'], W[pre + 'linears.2.bias']), h)
    else:
        kh, vh = _heads(k, h), _heads(v, h)
    x = dot_attention(qh, kh, vh, mask, p_drop).transpose(1, 2).contiguous().view(q.shape[0], -1, qh.shape[1] * qh.shape[3])
    if do_aoa:
        cat = torch.cat([x, q], -1)
        if aoa_drop is not None:
            cat = cat * aoa_drop
        x = F.glu(linear(cat, W[pre + 'aoa_layer.0.weight'], W[pre + 'aoa_layer.0.bias']), -1)
    return x.squeeze(1) if single else x


def aoa_prepare(W: Weights, fc: Tensor, att: Tensor, masks: Optional[Tensor], h: int, drop: Optional[Dict[str, Tensor]] = None):
    """``drop`` (train-mode replay): 'att' [B,R,H] after att_embed (AttModel.py:77-79); per refiner layer i 'ref_p%d' [B,h,R,R] on the
    attention probabilities, 'ref_aoa%d' [B,R,2H] on the AoA input, 'ref_sub%d' [B,R,H] in the SublayerConnection (TransformerModel.py:99-101)."""
    att, masks = clip_att(att, masks)
    x = torch.relu(linear(att, W['att_embed.0.weight'], W['att_embed.0.bias']))
    if drop is not None:
        x = x * drop['att']
    if masks is not None:
        x = x * masks.unsqueeze(-1).to(x)
    for i in range(6):
        pre = 'refiner.layers.%d.' % i
        y = _ln(W, pre + 'sublayer.0.norm.', x)
        # self_attn(x, x, x, mask): key = value = query source
        sub = aoa_mha(W, pre + 'self_attn.', y, y, y, masks, h, True, False, True, drop['ref_p%d' % i] if drop else None,
                      drop['ref_aoa%d' % i] if drop else None)
        x = x + (sub * drop['ref_sub%d' % i] if drop else sub)
    x = _ln(W, 'refiner.norm.', x)
    if masks is None:
        mean = x.mean(1)
    else:
        mean = (x * masks.unsqueeze(-1)).sum(1) / masks.unsqueeze(-1).sum(1)
    p_att = linear(x, W['ctx2att.weight'], W['ctx2att.bias'])
    return mean, x, p_att, masks


def aoa_core(W: Weights, xt: Tensor, mean: Tensor, att_e: Tensor, p_att: Tensor, state, masks, h: int, drop: Optional[Dict[str, Tensor]] = None):
    """``drop`` (one step of a train-mode replay): 'ctx' [N,H] on the carried context vector (ctx_drop, AoAModel.py:158-165), 'p' [N,h,1,R] on
    the attention probabilities, 'out' [N,H] on the returned output (out_drop, :186; the state keeps the un-dropped vector, :179)."""
    hs, cs = state                                  # [2, N, H]; hs[1] carries the previous context vector
    H = hs.shape[2]
    x1 = torch.cat([xt, mean + (hs[1] * drop['ctx'] if drop else hs[1])], 1)
    h_att, c_att = lstm_cell(x1, hs[0], cs[0], W['core.att_lstm.weight_ih'], W['core.att_lstm.weight_hh'], W['core.att_lstm.bias_ih'],
                             W['core.att_lstm.bias_hh'])
    # attention(h_att, p_att[..., :H], p_att[..., H:], mask) with signature (query, value, key)
    att = aoa_mha(W, 'core.attention.', h_att, p_att[..., H:], p_att[..., :H], masks, h, False, True, False, drop['p'] if drop else None)
    out = F.glu(linear(torch.cat([att, h_att], 1), W['core.att2ctx.0.weight'], W['core.att2ctx.0.bias']), -1)
    state = (torch.stack([h_att, out]), torch.stack([c_att, cs[1]]))
    return (out * drop['out'] if drop else out), state


# --------------------------------------------------------------------------------------------------
# family dispatch
# --------------------------------------------------------------------------------------------------

class Family:
    def __init__(self, name: str, W: Weights, seq_length: int, heads: int = 8):
        self.drop = None          # explicit dropout masks for a train-mode replay (UpDown, AoA)
        self.name = name
        self.W = W
        self.seq_length = seq_length
        if name == 'updown':
            self.num_layers = 2
            self.rnn_size = W['core.att_lstm.weight_hh'].shape[1]
            self.vocab1 = W['logit.weight'].shape[0]
        elif name == 'newfc':
            self.num_layers = 1
            self.rnn_size = W['_core.h2h.weight'].shape[1]
            self.vocab1 = W['logit.weight'].shape[0]
        elif name == 'aoa':
            self.num_layers = 2
            self.rnn_size = W['core.att_lstm.weight_hh'].shape[1]
            self.vocab1 = W['logit.weight'].shape[0]
            self.heads = heads
        elif name == 'transformer':
            self.vocab1 = W['model.generator.proj.weight'].shape[0]
            self.heads = heads
            self.n_layers = 1 + max(int(k.split('.')[3]) for k in W if k.startswith('model.decoder.layers.'))
        else:
            raise ValueError(name)

    def prepare(self, fc, att, masks=None):
        if self.name == 'updown':
            return updown_prepare(self.W, fc, att, masks, self.drop)
        if self.name == 'newfc':
            return newfc_prepare(self.W, fc, att, masks)
        if self.name == 'aoa':
            return aoa_prepare(self.W, fc, att, masks, self.heads, self.drop)
        return transformer_prepare(self.W, fc, att, masks, self.n_layers, self.heads, self.drop)

    def init_state(self, n: int):
        if self.name == 'transformer':
            return []
        z = torch.zeros(self.num_layers, n, self.rnn_size, dtype=self.W['logit.weight'].dtype)
        return (z, z.clone())

    def embed(self, it: Tensor) -> Tensor:
        if self.name in ('updown', 'aoa'):
            return torch.relu(self.W['embed.0.weight'][it])
        return self.W['embed.weight'][it]

    def logprobs_state(self, it, fc_e, att_e, p_att, masks, state, output_logsoftmax=True, t=None):
        if self.name == 'transformer':
            ys = it.unsqueeze(1) if len(state) == 0 else torch.cat([state[0][0], it.unsqueeze(1)], 1)
            out = transformer_decode(self.W, p_att, masks, ys, self.n_layers, self.heads)[:, -1]
            logits = linear(out, self.W['model.generator.proj.weight'], self.W['model.generator.proj.bias'])
            return (F.log_softmax(logits, dim=1) if output_logsoftmax else logits), [ys.unsqueeze(0)]
        xt = self.embed(it)
        if self.name == 'aoa':
            sd = None
            if self.drop is not None and t is not None:       # per-step masks: 'xt', 'ctx', 'p', 'out' are stacked over the steps
                xt = xt * self.drop['xt'][t]
                sd = {'ctx': self.drop['ctx'][t], 'p': self.drop['p'][t], 'out': self.drop['out'][t]}
            out, state = aoa_core(self.W, xt, fc_e, att_e, p_att, state, masks, self.heads, sd)
        elif self.name == 'updown':
            od = None
            if self.drop is not None and t is not None:
                xt = xt * self.drop['xt'][t]
                od = self.drop['out'][t]
            out, state = updown_core(self.W, xt, fc_e, att_e, p_att, state, masks, od)
        else:
            out, state = newfc_core(self.W, xt, fc_e, att_e, p_att, state, masks)
        logits = linear(out, self.W['logit.weight'], self.W['logit.bias'])
        return (F.log_softmax(logits, dim=1) if output_logsoftmax else logits), state


# --------------------------------------------------------------------------------------------------
# beam search
# --------------------------------------------------------------------------------------------------

def _length_penalty(cfg: str):
    if cfg == '':
        return lambda length, lp: lp
    kind, alpha = cfg.split('_')
    alpha = float(alpha)
    if kind == 'wu':
        return lambda length, lp: lp / (((5 + length) ** alpha) / ((5 + 1) ** alpha))
    if kind == 'avg':
        return lambda length, lp: lp / length
    raise ValueError(cfg)


def beam_search(fam: Family, init_state, init_logprobs: Tensor, fc_e, att_e, p_att, masks, beam_size: int,
                length_penalty: str = '', temperature: float = 1.0, eos_idx: int = 0, record_margin: Optional[list] = None,
                margin_rows: Optional[list] = None):
    """Classical batched beam search, one group.  Returns list[B] of list[<=beam] records.

    State/feature rows are image-major: row i*beam+j is beam j of image i.  The first step works on B rows
    (one live beam per image).  A beam that emits EOS, or any beam at the last step, is recorded and its
    running sum is lowered by 1000 -- but it stays in the beam and keeps being expanded, fed token 0.
    """
    pen = _length_penalty(length_penalty)
    B, V1 = init_logprobs.shape
    T = fam.seq_length
    seqs = torch.zeros(B, beam_size, 0, dtype=torch.long)
    hist = torch.zeros(B, beam_size, 0, V1)
    sums = torch.zeros(B, beam_size)
    state = [s.clone() for s in init_state]
    logprobs = init_logprobs.clone()
    done: List[List[dict]] = [[] for _ in range(B)]
    for t in range(T):
        lp = logprobs.reshape(B, -1, V1)                      # [B, live, V1]
        live = lp.shape[1]
        cand = (sums[:, :live].unsqueeze(-1) + lp).reshape(B, -1)
        ys, ix = torch.sort(cand, -1, True)
        if record_margin is not None:
            record_margin.append(float((ys[:, :beam_size] - ys[:, 1:beam_size + 1]).min()))
        if margin_rows is not None:          # per-image smallest gap among the top beam_size + 1 candidates of this step
            gaps = ys[:, :beam_size] - ys[:, 1:beam_size + 1]
            gaps = torch.where(ys[:, :beam_size] > -500.0, gaps, torch.full_like(gaps, 1e9))     # ended beams (sum - 1000) tie freely: ignore
            margin_rows.append(gaps.min(1).values.clone())
        ys, ix = ys[:, :beam_size], ix[:, :beam_size]
        parent = ix // V1
        word = ix % V1
        rows = (parent + torch.arange(B).unsqueeze(-1) * live).reshape(-1)
        if t > 0:
            seqs = seqs.gather(1, parent.unsqueeze(-1).expand_as(seqs))
            hist = hist.gather(1, parent.unsqueeze(-1).unsqueeze(-1).expand_as(hist))
        seqs = torch.cat([seqs, word.unsqueeze(-1)], -1)
        sums = sums[:, :live].gather(1, parent) + lp.reshape(B, -1).gather(1, ix)
        hist = torch.cat([hist, lp.gather(1, parent.unsqueeze(-1).expand(-1, -1, V1)).unsqueeze(2)], 2)
        state = [s[:, rows] for s in state]
        ended = (word == eos_idx) if t < T - 1 else torch.ones_like(word, dtype=torch.bool)
        for b in range(B):
            for v in range(beam_size):
                if ended[b, v]:
                    done[b].append({'seq': seqs[b, v].clone(), 'logps': hist[b, v].clone(),
                                    'unaug_p': float(hist[b, v].sum()), 'p': pen(t + 1, float(sums[b, v]))})
        sums = sums - 1000.0 * ended.to(sums)
        it = word.reshape(-1)
        logprobs, state = fam.logprobs_state(it, fc_e, att_e, p_att, masks, state)
        state = list(state)
        logprobs = F.log_softmax(logprobs / temperature, dim=-1)
    return [sorted(d, key=lambda r: -r['p'])[:beam_size] for d in done]


def sample_beam(fam: Family, fc: Tensor, att: Tensor, masks: Optional[Tensor] = None, beam_size: int = 5, sample_n: int = 1,
                length_penalty: str = '', record_margin: Optional[list] = None, margin_rows: Optional[list] = None):
    assert sample_n in (1, beam_size)
    B = fc.shape[0]
    T, V1 = fam.seq_length, fam.vocab1
    fc_e, att_e, p_att, masks = fam.prepare(fc, att, masks)
    state = fam.init_state(B)
    it = torch.zeros(B, dtype=torch.long)
    logprobs, state = fam.logprobs_state(it, fc_e, att_e, p_att, masks, state)
    fc_r, att_r, p_att_r, masks_r = (repeat_rows(x, beam_size) for x in (fc_e, att_e, p_att, masks))
    done = beam_search(fam, state, logprobs, fc_r, att_r, p_att_r, masks_r, beam_size, length_penalty, record_margin=record_margin,
                       margin_rows=margin_rows)
    seq = torch.zeros(B * sample_n, T, dtype=torch.long)
    seq_lp = torch.zeros(B * sample_n, T, V1, dtype=fc.dtype)
    for k in range(B):
        for n in range(sample_n):
            rec = done[k][n]
            L = rec['seq'].shape[0]
            seq[k * sample_n + n, :L] = rec['seq']
            seq_lp[k * sample_n + n, :L] = rec['logps']
    return seq, seq_lp, done


# --------------------------------------------------------------------------------------------------
# greedy / multinomial sampling
# --------------------------------------------------------------------------------------------------

def sample(fam: Family, fc: Tensor, att: Tensor, masks: Optional[Tensor] = None, sample_method: str = 'greedy',
           sample_n: int = 1, temperature: float = 1.0, forced_tokens: Optional[Tensor] = None, eos_idx: int = 0,
           record_margin: Optional[list] = None):
    """Returns (seq [N,T] int64, seqLogprobs [N,T,V1]).  ``forced_tokens`` replays a given sample (used to compare
    log-prob rows when the sampler's random stream differs)."""
    B = fc.shape[0]
    N = B * sample_n
    T, V1 = fam.seq_length, fam.vocab1
    fc_e, att_e, p_att, masks = fam.prepare(fc, att, masks)
    fc_e, att_e, p_att, masks = (repeat_rows(x, sample_n) for x in (fc_e, att_e, p_att, masks))
    state = fam.init_state(N)
    seq = torch.zeros(N, T, dtype=torch.long)
    seq_lp = torch.zeros(N, T, V1, dtype=fc.dtype)
    it = torch.zeros(N, dtype=torch.long)
    unfinished = None
    for t in range(T):
        logprobs, state = fam.logprobs_state(it, fc_e, att_e, p_att, masks, state, t=t)
        if forced_tokens is not None:
            it = forced_tokens[:, t].clone()
        elif sample_method == 'greedy':
            top2 = logprobs.topk(2, dim=1).values
            if record_margin is not None:
                live = torch.ones(N, dtype=torch.bool) if unfinished is None else unfinished
                if bool(live.any()):
                    record_margin.append(float((top2[:, 0] - top2[:, 1])[live].min()))
            it = logprobs.argmax(1)
        else:
            # the temperature only shapes the sampling distribution; the stored row stays unscaled
            it = torch.distributions.Categorical(logits=logprobs / temperature).sample()
        if t == 0:
            unfinished = it != eos_idx
        else:
            it = it * unfinished.to(it)
            logprobs = logprobs * unfinished.unsqueeze(1).to(logprobs)
            unfinished = unfinished & (it != eos_idx)
        seq[:, t] = it
        seq_lp[:, t] = logprobs
        if int(unfinished.sum()) == 0:
            break
    return seq, seq_lp


# --------------------------------------------------------------------------------------------------
# teacher forcing and the SCST criterion
# --------------------------------------------------------------------------------------------------

def forward_teacher(fam: Family, fc: Tensor, att: Tensor, seq: Tensor, masks: Optional[Tensor] = None, pad_keys_masked: bool = True):
    """``pad_keys_masked=False`` (transformer): causal mask only -- what core() applies while sampling (TransformerModel.py:351-363), so the one-pass
    result equals the step-by-step log-probs of a sampled prefix."""
    B = fc.shape[0]
    if seq.dim() == 3:
        seq = seq.reshape(-1, seq.shape[2])
    spi = seq.shape[0] // B
    N = B * spi
    if fam.name == 'transformer':        # one parallel pass with the pad/eos + causal mask (TransformerModel.py:324-348)
        _, _, memory, m3 = fam.prepare(fc, att, masks)
        memory, m3 = repeat_rows(memory, spi), repeat_rows(m3, spi)
        seq_mask = (seq != 0)
        seq_mask[:, 0] = True
        t = seq.shape[1]
        tgt_mask = torch.tril(torch.ones(1, t, t, dtype=torch.bool))
        if pad_keys_masked:
            tgt_mask = seq_mask.unsqueeze(-2) & tgt_mask
        out = transformer_decode(fam.W, memory, m3, seq, fam.n_layers, fam.heads, tgt_mask, fam.drop)
        return F.log_softmax(linear(out, fam.W['model.generator.proj.weight'], fam.W['model.generator.proj.bias']), dim=-1)
    fc_e, att_e, p_att, masks = fam.prepare(fc, att, masks)
    fc_e, att_e, p_att, masks = (repeat_rows(x, spi) for x in (fc_e, att_e, p_att, masks))
    state = fam.init_state(N)
    out = torch.zeros(N, seq.shape[1], fam.vocab1, dtype=fc.dtype)
    for i in range(seq.shape[1]):
        if i >= 1 and int(seq[:, i].sum()) == 0:
            break
        lp, state = fam.logprobs_state(seq[:, i].clone(), fc_e, att_e, p_att, masks, state, t=i if fam.drop is not None else None)
        out[:, i] = lp
    return out


def reward_criterion(logprobs: Tensor, seq: Tensor, reward: Tensor, reduction: str = 'mean') -> Tensor:
    N, L = seq.shape
    picked = logprobs.gather(2, seq.unsqueeze(2)).squeeze(2)
    mask = (seq > 0).to(picked)
    mask = torch.cat([torch.ones(N, 1), mask[:, :-1]], 1)
    out = -picked * reward * mask
    if reduction == 'none':
        return out.sum(1) / mask.sum(1)
    return out.sum() / mask.sum()


def language_model_criterion(logprobs: Tensor, target: Tensor, mask: Tensor, reduction: str = 'mean') -> Tensor:
    """captioning/modules/losses.py:204-225: masked NLL of the targets; target/mask are cut to the log-prob width."""
    if target.dim() == 3:
        target, mask = target.reshape(-1, target.shape[2]), mask.reshape(-1, mask.shape[2])
    L = logprobs.shape[1]
    target, mask = target[:, :L], mask[:, :L].to(logprobs)
    out = -logprobs.gather(2, target.unsqueeze(2)).squeeze(2) * mask
    if reduction == 'none':
        return out.sum(1) / mask.sum(1)
    return out.sum() / mask.sum()


def label_smoothing_loss(logprobs: Tensor, target: Tensor, mask: Tensor, smoothing: float, reduction: str = 'mean') -> Tensor:
    """captioning/modules/losses.py:228-265: KLDiv(logp, smoothed one-hot) summed over the vocabulary, masked; the smoothed
    distribution puts ``smoothing / (V1 - 1)`` everywhere and ``1 - smoothing`` on the target (:251-253)."""
    N, L, V1 = logprobs.shape
    if target.dim() == 3:
        target, mask = target.reshape(-1, target.shape[2]), mask.reshape(-1, mask.shape[2])
    target, mask = target[:, :L].reshape(-1), mask[:, :L].reshape(-1).to(logprobs)
    lp = logprobs.reshape(-1, V1)
    dist = torch.full_like(lp, smoothing / (V1 - 1))
    dist.scatter_(1, target.unsqueeze(1), 1.0 - smoothing)
    kl = (dist * (torch.log(dist) - lp)).sum(1) * mask
    if reduction == 'none':
        return kl.view(N, L).sum(1) / mask.view(N, L).sum(1)
    return kl.sum() / mask.sum()


def new_self_critical_loss(logprobs: Tensor, seq: Tensor, scores: Tensor, sample_n: int, reduction: str = 'mean') -> Tensor:
    """StructureLosses, loss_type 'new_self_critical' (captioning/modules/losses.py:46-67, :168-187): ``scores`` [N] are the CIDEr-D
    values of get_scores cast to the log-prob dtype; each sample's weight is its score minus the mean of the image's other samples."""
    N, L = seq.shape
    mask = torch.cat([torch.ones(N, 1), (seq > 0).to(logprobs)[:, :-1]], 1)
    sc = scores.to(logprobs).view(-1, sample_n)
    sc = sc - (sc.sum(1, keepdim=True) - sc) / (sample_n - 1)
    picked = logprobs.gather(2, seq.unsqueeze(2)).squeeze(2)
    out = -picked * mask * sc.reshape(-1, 1)
    if reduction == 'none':
        return out.sum(1) / mask.sum(1)
    return out.sum() / mask.sum()


def reward_criterion_grad(seq: Tensor, reward: Tensor, V1: int) -> Tensor:
    """d(loss_mean)/d(logprobs): -reward*mask/sum(mask) scattered at the sampled ids."""
    N, L = seq.shape
    mask = torch.cat([torch.ones(N, 1), (seq > 0).float()[:, :-1]], 1)
    g = torch.zeros(N, L, V1)
    g.scatter_(2, seq.unsqueeze(2), (-(reward * mask) / mask.sum()).unsqueeze(2))
    return g


# --------------------------------------------------------------------------------------------------
# synthetic weights / inputs: the seeded generators live in the package (imagecaptioning.pytorch_b200.synthetic) because bench.py's
# GPU arm needs them without importing the oracle; re-exported here for the tests and the golden generator.
# --------------------------------------------------------------------------------------------------
from imagecaptioning.pytorch_b200.synthetic import make_inputs, make_weights      # noqa: E402,F401
