"""Plain-PyTorch restatement of Att2in2Model (captioning/models/AttModel.py:754-790, 854-859), the checker of the engine's Att2in2 family.

It plugs into the oracle's decode functions (co.sample, co.sample_beam, co.forward_teacher, dbs_oracle.diverse_sample_beam) as a Family:
* the prologue is AttModel._prepare_feature with fc_embed the identity: att_embed (Linear + ReLU, optional train-mode dropout mask, the
  region mask of pack_wrapper) and ctx2att;
* the core is co.additive_attention on the PREVIOUS hidden state followed by co.maxout_lstm.  Att2in2's gate sums
  i2h(xt) + h2h(h) + [0 | a2c(att_res)] are NewFC's maxout sums with the input [xt | att_res] and an i2h whose rows 3H..5H are extended
  by a2c (its bias by a2c's bias), so the maxout cell is reused unchanged.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle import caption_oracle as co


def maxout_weights(W):
    """The co.maxout_lstm weight dict of an Att2in2 core: input [xt | att_res]."""
    i2h_w, i2h_b, a2c_w, a2c_b = W['core.i2h.weight'], W['core.i2h.bias'], W['core.a2c.weight'], W['core.a2c.bias']
    H = a2c_w.shape[1]
    pad_w = torch.cat([torch.zeros(3 * H, H, dtype=a2c_w.dtype), a2c_w], 0)
    pad_b = torch.cat([torch.zeros(3 * H, dtype=a2c_b.dtype), a2c_b], 0)
    return {'_core.i2h.weight': torch.cat([i2h_w, pad_w], 1), '_core.i2h.bias': i2h_b + pad_b,
            '_core.h2h.weight': W['core.h2h.weight'], '_core.h2h.bias': W['core.h2h.bias']}


def att2in2_core(W, xt, att_e, p_att, state, masks=None, out_drop=None):
    h, c = state                                   # [1, N, H]
    att_res = co.additive_attention(W, h[-1], att_e, p_att, masks)
    out, state = co.maxout_lstm(maxout_weights(W), torch.cat([xt, att_res], 1), state)
    return (out if out_drop is None else out * out_drop), state


class Att2in2Family(co.Family):
    """co.Family for 'att2in2'.  ``drop`` (train-mode replay) carries {'att': [B,R,H], 'xt': [T,N,E], 'out': [T,N,H]}."""

    def __init__(self, W, seq_length: int):
        self.drop = None
        self.name = 'att2in2'
        self.W = W
        self.seq_length = seq_length
        self.num_layers = 1
        self.rnn_size = W['core.h2h.weight'].shape[1]
        self.vocab1 = W['logit.weight'].shape[0]

    def prepare(self, fc, att, masks=None):
        att, masks = co.clip_att(att, masks)
        att_e = torch.relu(co.linear(att, self.W['att_embed.0.weight'], self.W['att_embed.0.bias']))
        if self.drop is not None:
            att_e = att_e * self.drop['att']
        if masks is not None:
            att_e = att_e * masks.unsqueeze(-1).to(att_e)
        return fc, att_e, co.linear(att_e, self.W['ctx2att.weight'], self.W['ctx2att.bias']), masks

    def embed(self, it):
        return torch.relu(self.W['embed.0.weight'][it])

    def logprobs_state(self, it, fc_e, att_e, p_att, masks, state, output_logsoftmax=True, t=None):
        xt = self.embed(it)
        od = None
        if self.drop is not None and t is not None:
            xt = xt * self.drop['xt'][t]
            od = self.drop['out'][t]
        out, state = att2in2_core(self.W, xt, att_e, p_att, state, masks, od)
        logits = co.linear(out, self.W['logit.weight'], self.W['logit.bias'])
        return (F.log_softmax(logits, dim=1) if output_logsoftmax else logits), state
