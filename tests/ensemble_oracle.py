"""Plain-PyTorch restatement of AttEnsemble (captioning/models/AttEnsemble.py), the checker of the engine's test-time ensemble.

``EnsembleFamily`` plugs into the oracle's decode loops as one Family:
* prepare runs every member's own _prepare_feature (AttEnsemble._prepare_feature :64-65) and hands the decode loops the image index of each
  row in place of the features, so their row repetition (repeat_tensors) repeats the index and each member looks its features up per row;
* the state is the members' states concatenated (pack_state :34-36), which the beam loops reorder row-wise like a single model's;
* the decode loops are co.sample / co.forward_teacher and, for beam search with its decode options, dbs_oracle.diverse_sample_beam
  with group_size 1 (CaptionModel.beam_search);
* logprobs_state runs each member's core, takes softmax of its logits and mixes them in the reference's fp32 order,
  stack -> * weights -> / weights.sum() -> sum over members -> log (get_logprobs_state :50-58).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle import caption_oracle as co
import att2in2_oracle as ao
import dbs_oracle


def member_family(name, W, seq_length, heads=8):
    return ao.Att2in2Family(W, seq_length) if name == 'att2in2' else co.Family(name, W, seq_length, heads=heads)


def _rows(x, idx):
    return x[idx] if torch.is_tensor(x) else x


class EnsembleFamily:
    def __init__(self, members, weights=None):
        self.members = list(members)
        self.weights = torch.tensor(weights or [1.0] * len(self.members))
        self.name = 'ensemble'
        self.drop = None
        self.seq_length = self.members[0].seq_length
        self.vocab1 = self.members[0].vocab1
        self._feats = None
        self._lens = None

    def prepare(self, fc, att, masks=None):
        self._feats = [m.prepare(fc, att, masks) for m in self.members]
        _, masks = co.clip_att(att, masks)
        idx = torch.arange(fc.shape[0])
        return idx, idx, idx, masks

    def init_state(self, n):
        states = [list(m.init_state(n)) for m in self.members]
        self._lens = [len(s) for s in states]
        return sum(states, [])

    def mix(self, logits):
        """log( sum_k softmax(z_k) w_k / sum w ) of the members' raw logits [N, V1] each."""
        return torch.stack([F.softmax(z, dim=1) for z in logits], 2).mul(self.weights).div(self.weights.sum()).sum(-1).log()

    def logprobs_state(self, it, fc_e, att_e, p_att, masks, state, output_logsoftmax=True, t=None):
        assert output_logsoftmax, 'AttEnsemble always returns log-probabilities'
        idx = fc_e                                   # image of each row
        logits, new_state, i = [], [], 0
        for m, f, n in zip(self.members, self._feats, self._lens):
            z, st = m.logprobs_state(it, _rows(f[0], idx), _rows(f[1], idx), _rows(f[2], idx), masks, tuple(state[i:i + n]), output_logsoftmax=False)
            logits.append(z)
            new_state += list(st)
            i += n
        return self.mix(logits), new_state


# --------------------------------------------------------------------------------------------------
# the cases of tests/golden/ensemble_small.npz (tests/make_ensemble_golden.py), shared by the CPU and GPU tests
# --------------------------------------------------------------------------------------------------

def labels(B, T, V, seed):
    """Teacher-forcing labels [B, 2, T + 2] (seq_per_img 2, <bos> first, zero padded after a random length)."""
    g = torch.Generator().manual_seed(seed)
    lab = torch.randint(1, V + 1, (B * 2, T + 2), generator=g)
    lens = torch.randint(3, T + 1, (B * 2,), generator=g)
    lab[:, 0] = 0
    for i in range(B * 2):
        lab[i, int(lens[i]) + 1:] = 0
    return lab.reshape(B, 2, T + 2)


def case_masks(B, R):
    masks = torch.ones(B, R)
    masks[1, 5:] = 0
    masks[3, 3:] = 0
    return masks


def mix_weights(meta, mix, wname):
    w = meta['weights'][wname]
    return None if w is None else w[str(len(meta['mixes'][mix]))]


def member_weight_dicts(meta, mix):
    c = meta['cfg']
    return [(f, co.make_weights(f, c['V'], c['E'], c['H'], c['A'], c['F_fc'], c['F_att'], seed=s, logit_scale=meta['logit_scale']))
            for f, s in meta['mixes'][mix]]


def oracle_for(meta, mix, wname):
    members = [member_family(f, W, meta['cfg']['T'], heads=meta['aoa_heads']) for f, W in member_weight_dicts(meta, mix)]
    return EnsembleFamily(members, mix_weights(meta, mix, wname))


def run_oracle(fam, fc, att, meta, opts, masked, margins=None):
    """The reference's outputs of one golden case, restated: {'out'} (teacher forcing) or {'seq', 'logprobs'[, 'done']}.  ``margins``
    (list) receives the per-image smallest winner / runner-up gap of every step (greedy and beam search)."""
    masks = case_masks(meta['B'], meta['R']) if masked else None
    if opts == 'teacher':
        c = meta['cfg']
        return {'out': co.forward_teacher(fam, fc, att, labels(meta['B'], c['T'], c['V'], meta['label_seed']), masks)}
    if opts.get('beam_size', 1) > 1:
        seq, lp, done = dbs_oracle.diverse_sample_beam(fam, fc, att, masks, beam_size=opts['beam_size'], group_size=1,
                                                       length_penalty=opts.get('length_penalty', ''),
                                                       decoding_constraint=bool(opts.get('decoding_constraint', 0)), margin_rows=margins)
        return {'seq': seq, 'logprobs': lp, 'done': done}
    rec = [] if margins is not None else None
    seq, lp = co.sample(fam, fc, att, masks, record_margin=rec)
    if margins is not None:
        margins.extend(torch.full((meta['B'],), m) for m in rec)
    return {'seq': seq, 'logprobs': lp}
