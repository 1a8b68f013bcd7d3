"""Plain-PyTorch restatement of NewFCModel in train mode (captioning/models/AttModel.py:904-945 with FCModel.LSTMCore, FCModel.py:13-42),
the checker of the engine's fused NewFC training steps.

It plugs into the oracle's decode functions (co.sample, co.forward_teacher) as a co.Family built from co.newfc_prepare, co.maxout_lstm and
co.newfc_core: a zero state first consumes fc_embed(fc) (the image step; its output is dropped), then the words.  ``drop`` (a train-mode
replay) carries the masks of the model's only dropout site, the core output before ``logit``: {'out': [T, N, H]}.  The region features are
never read, so ``att`` may have any shape, [B, 0, 0] included.
"""
from __future__ import annotations

import torch.nn.functional as F

from oracle import caption_oracle as co


class NewFCFamily(co.Family):
    """co.Family('newfc') with the core-output dropout of a train-mode step."""

    def __init__(self, W, seq_length: int):
        super().__init__('newfc', W, seq_length)

    def logprobs_state(self, it, fc_e, att_e, p_att, masks, state, output_logsoftmax=True, t=None):
        out, state = co.newfc_core(self.W, self.embed(it), fc_e, att_e, p_att, state, masks)
        if self.drop is not None and t is not None:
            out = out * self.drop['out'][t]
        logits = co.linear(out, self.W['logit.weight'], self.W['logit.bias'])
        return (F.log_softmax(logits, dim=1) if output_logsoftmax else logits), state
