"""Plain-PyTorch restatement of diverse beam search (CaptionModel.beam_search with group_size > 1, CaptionModel.py:35-209), the checker of
the engine's diverse beam search.

It follows the reference step for step, with one repair: add_diversity calls ``self.repeat_tensor(bdash, change)`` (CaptionModel.py:53),
a method that does not exist, so the reference raises AttributeError at the first step of group 1 past its first position.  The intended
function is captioning/models/utils.py:repeat_tensors, which repeats each image's penalty row once per beam of the group; that is what
this restatement does.  Everything else is the reference's behaviour, including its quirks:

* every group starts from the same <bos>-step log-probs (one row per image, a single log_softmax) and group g starts g steps late;
* ``logps`` holds the un-augmented (edited, not penalised) rows; running sums and the record scores ``p`` accumulate the penalised ones;
* ``done_beams[i]`` is each group's records sorted by ``p`` and cut to bdash, concatenated in group order (not globally sorted);
* with sample_n == bdash, AttModel._sample_beam fills only rows 0 .. B-1 of ``seq`` (done_beams[k][0]); the other rows stay pad.
"""
from __future__ import annotations

from typing import List, Optional

import torch
import torch.nn.functional as F

from oracle import caption_oracle as co


def diverse_sample_beam(fam: co.Family, fc, att, masks=None, beam_size: int = 4, group_size: int = 2, diversity_lambda: float = 0.5,
                        sample_n: int = 1, length_penalty: str = '', temperature: float = 1.0, decoding_constraint: bool = False,
                        eos_idx: int = 0, margin_rows: Optional[list] = None):
    """Returns (seq [B*sample_n, T], seq_logprobs [B*sample_n, T, V+1], done_beams).  margin_rows (optional list) receives, per group step,
    each image's smallest gap among the group's top bdash + 1 candidates (ended beams excluded): how far each decision is from a tie."""
    G = group_size
    assert beam_size % G == 0
    bdash = beam_size // G
    assert sample_n in (1, bdash)
    pen = co._length_penalty(length_penalty)
    B = fc.shape[0]
    T, V1 = fam.seq_length, fam.vocab1
    fc_e, att_e, p_att, masks_ = fam.prepare(fc, att, masks)
    init_state = fam.init_state(B)
    init_lp, init_state = fam.logprobs_state(torch.zeros(B, dtype=torch.long), fc_e, att_e, p_att, masks_, init_state)
    feats = [co.repeat_rows(x, bdash) for x in (fc_e, att_e, p_att, masks_)]      # every row of a group carries its image's features
    seqs = [torch.zeros(B, bdash, 0, dtype=torch.long) for _ in range(G)]
    hist = [torch.zeros(B, bdash, 0, V1) for _ in range(G)]
    sums = [torch.zeros(B, bdash) for _ in range(G)]
    states = [[s.clone() for s in init_state] for _ in range(G)]
    logprobs = [init_lp.clone() for _ in range(G)]
    done: List[List[List[dict]]] = [[[] for _ in range(G)] for _ in range(B)]
    for t in range(T + G - 1):
        for g in range(G):
            lt = t - g
            if lt < 0 or lt > T - 1:
                continue
            lp = logprobs[g]
            if decoding_constraint and lt > 0:
                lp = lp.clone()
                lp.scatter_(1, seqs[g][:, :, lt - 1].reshape(-1, 1), float('-inf'))
            unaug = lp.clone()
            if g > 0:           # add_diversity: the earlier groups' words at this position, in their current beams
                change = torch.zeros(B, V1)
                for pg in range(g):
                    prev = seqs[pg][:, :, lt]
                    for j in range(bdash):
                        change.scatter_add_(1, prev[:, j:j + 1], torch.ones(B, 1))
                lp = lp - (change if lt == 0 else co.repeat_rows(change, bdash)) * diversity_lambda
            lpr = lp.reshape(B, -1, V1)
            live = lpr.shape[1]
            cand = (sums[g][:, :live].unsqueeze(-1) + lpr).reshape(B, -1)
            ys, ix = torch.sort(cand, stable=True, dim=-1, descending=True)
            if margin_rows is not None:
                gaps = ys[:, :bdash] - ys[:, 1:bdash + 1]
                gaps = torch.where(ys[:, :bdash] > -500.0, gaps, torch.full_like(gaps, 1e9))
                margin_rows.append(gaps.min(1).values.clone())
            ys, ix = ys[:, :bdash], ix[:, :bdash]
            parent, word = ix // V1, ix % V1
            rows = (parent + torch.arange(B).unsqueeze(-1) * live).reshape(-1)
            if lt > 0:
                seqs[g] = seqs[g].gather(1, parent.unsqueeze(-1).expand_as(seqs[g]))
                hist[g] = hist[g].gather(1, parent.unsqueeze(-1).unsqueeze(-1).expand_as(hist[g]))
            seqs[g] = torch.cat([seqs[g], word.unsqueeze(-1)], -1)
            sums[g] = sums[g][:, :live].gather(1, parent) + lpr.reshape(B, -1).gather(1, ix)
            hist[g] = torch.cat([hist[g], unaug.reshape(B, -1, V1).gather(1, parent.unsqueeze(-1).expand(-1, -1, V1)).unsqueeze(2)], 2)
            states[g] = [s[:, rows] for s in states[g]]
            ended = (word == eos_idx) if lt < T - 1 else torch.ones_like(word, dtype=torch.bool)
            for b in range(B):
                for v in range(bdash):
                    if ended[b, v]:
                        done[b][g].append({'seq': seqs[g][b, v].clone(), 'logps': hist[g][b, v].clone(),
                                           'unaug_p': float(hist[g][b, v].sum()), 'p': pen(lt + 1, float(sums[g][b, v]))})
            sums[g] = sums[g] - 1000.0 * ended.to(sums[g])
            out, st = fam.logprobs_state(word.reshape(-1), *feats, states[g])
            states[g] = list(st)
            logprobs[g] = F.log_softmax(out / temperature, dim=-1)
    done_beams = [sum([sorted(done[b][g], key=lambda r: -r['p'])[:bdash] for g in range(G)], []) for b in range(B)]
    seq = torch.zeros(B * sample_n, T, dtype=torch.long)
    seq_lp = torch.zeros(B * sample_n, T, V1)
    for k in range(B):
        rec = done_beams[k][0]
        L = rec['seq'].shape[0]
        seq[k, :L] = rec['seq']
        seq_lp[k, :L] = rec['logps']
    return seq, seq_lp, done_beams


def beams_to_arrays(done_beams, n, T):
    """done_beams -> (seq [B, n, T] int64, len [B, n], p [B, n] float64)."""
    import numpy as np
    B = len(done_beams)
    seqs, lens, ps = np.zeros((B, n, T), np.int64), np.zeros((B, n), np.int64), np.zeros((B, n), np.float64)
    for i, lst in enumerate(done_beams):
        for j, rec in enumerate(lst):
            L = rec['seq'].shape[0]
            seqs[i, j, :L] = rec['seq'].numpy()
            lens[i, j] = L
            ps[i, j] = rec['p']
    return seqs, lens, ps
