"""AttModel's output head for logit_layers = k > 1 (captioning/models/AttModel.py:87-92), wrapped around any oracle Family.

The head is k - 1 hidden [Linear(H, H), ReLU, Dropout(0.5)] blocks ahead of the vocabulary Linear, applied to the core's output at every
step (get_logprobs_state :166-176); the state carried to the next step is the core's, not the head's.  ``HeadFamily`` runs the wrapped
family with an identity vocabulary layer (so its "logits" are the core output, exactly: x I^T + 0 rounds nothing), then the head.  It plugs
into the oracle's decode loops (co.sample, co.sample_beam, co.forward_teacher, dbs_oracle.diverse_sample_beam) and into EnsembleFamily as
a member.  Dropout is a train-mode op: the decode loops apply none; ``head_drop`` (a train-mode replay) holds the fused steps' masks
of hidden layer i at position t, [k - 1][T, N, H] (capb200_dropout_mask site 200 + i, step t).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle import caption_oracle as co


def head_layers(W):
    """[(weight, bias)] of W's logit head in order: the hidden layers, then the vocabulary Linear."""
    idx = sorted({int(k.split('.')[1]) for k in W if k.startswith('logit.') and k.count('.') == 2})
    return [(W['logit.%d.weight' % i], W['logit.%d.bias' % i]) for i in idx]


HEAD_DROP_SITE = 200


def apply_head(layers, x, masks=None):
    for i, (w, b) in enumerate(layers[:-1]):
        x = torch.relu(co.linear(x, w, b))
        if masks is not None:
            x = x * masks[i]
    return co.linear(x, *layers[-1])


class HeadFamily:
    """``make_family(W_core, *args, **kwargs)`` builds the wrapped family (co.Family's name argument bound, or Att2in2Family)."""

    def __init__(self, make_family, W, *args, **kwargs):
        self.layers = head_layers(W)
        H = self.layers[0][0].shape[1]
        dt = self.layers[-1][0].dtype
        core_W = {k: v for k, v in W.items() if not k.startswith('logit.')}
        core_W['logit.weight'], core_W['logit.bias'] = torch.eye(H, dtype=dt), torch.zeros(H, dtype=dt)
        self.base = make_family(core_W, *args, **kwargs)
        self.W = W
        self.vocab1 = self.layers[-1][0].shape[0]
        self.head_drop = None

    @property
    def drop(self):          # what the decode loops test before they pass the position t (co.forward_teacher)
        base = self.base.drop
        return base if base is not None or self.head_drop is None else {}

    @drop.setter
    def drop(self, value):
        self.base.drop = value

    def __getattr__(self, name):                  # prepare, init_state, embed, name, seq_length, drop: the wrapped family's
        return getattr(self.__dict__['base'], name)

    def logprobs_state(self, it, fc_e, att_e, p_att, masks, state, output_logsoftmax=True, t=None):
        out, state = self.base.logprobs_state(it, fc_e, att_e, p_att, masks, state, output_logsoftmax=False, t=t)
        hm = None if self.head_drop is None or t is None else [m[t] for m in self.head_drop]
        logits = apply_head(self.layers, out, hm)
        return (F.log_softmax(logits, dim=1) if output_logsoftmax else logits), state


def family(name, W, seq_length, heads=8):
    """The oracle family of an engine family ('updown', 'att2in2', 'newfc', 'aoa') with W's logit head."""
    import att2in2_oracle as ao
    if name == 'att2in2':
        return HeadFamily(ao.Att2in2Family, W, seq_length)
    return HeadFamily(lambda w, T: co.Family(name, w, T, heads=heads), W, seq_length)
