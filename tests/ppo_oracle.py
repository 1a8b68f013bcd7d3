"""PPO restated in plain torch (losses.py:267-357, PPOLoss.forward), the oracle the PPO tests hold the fused steps to.

    ppo_loss(lp, lo, seq, scores, n, cliprange, kl_coef, reduction) -> {'loss', 'pg_loss', 'kl_loss', 'clipfrac', 'reward'}

lp [N, T, V+1] are the new policy's sampled log-probs (differentiable), lo the old policy's teacher-forced log-probs over [0, seq[:, :-1]],
scores [N] the rewarded caption scores (n samples per image).  The clipped surrogate takes the unclamped branch inside the clip range and,
outside it, whichever branch is larger -- the branch torch.maximum hands the gradient to.
"""
from __future__ import annotations

import torch


def token_mask(seq):
    """1 for every word up to and including the first EOS (losses.py:296-297)."""
    live = (seq > 0).to(torch.float64)
    return torch.cat([torch.ones_like(live[:, :1]), live[:, :-1]], 1)


def old_policy_input(seq):
    """The old policy's teacher-forced input: BOS, then the sampled words shifted by one (losses.py:319)."""
    return torch.cat([torch.zeros_like(seq[:, :1]), seq[:, :-1]], 1)


def ppo_loss(lp, lo, seq, scores, n, cliprange=0.2, kl_coef=0.02, reduction='mean', adv=None):
    """``adv`` [N], when given, replaces the leave-one-out advantage of ``scores`` (which may then be None): the rows of a step taken apart
    from their image's other samples."""
    mask = token_mask(seq).to(lp.dtype)
    if adv is None:
        reward = scores.to(lp.dtype).reshape(-1, n)
        adv = (reward - (reward.sum(1, keepdim=True) - reward) / (n - 1)).reshape(-1, 1)
    else:
        reward = None
        adv = adv.to(lp.dtype).reshape(-1, 1)
    idx = seq.unsqueeze(2)
    ratio = torch.exp(lp.gather(2, idx).squeeze(2) - lo.gather(2, idx).squeeze(2))
    clamped = ratio.clamp(1.0 - cliprange, 1.0 + cliprange)
    unclamped = (ratio == clamped) | (-adv * ratio > -adv * clamped)
    pg = torch.where(unclamped, -adv * ratio, -adv * clamped)
    kl = (lo.exp() * (lo - lp)).sum(2)
    clip = ((ratio - 1.0).abs() > cliprange).to(lp.dtype)
    total = mask.sum()
    out = {'reward': reward, 'pg_loss': (pg * mask).sum() / total, 'kl_loss': (kl * mask).sum() / total, 'clipfrac': (clip * mask).sum() / total}
    if reduction == 'none':
        out['loss'] = ((pg + kl_coef * kl) * mask).sum(1) / mask.sum(1)
    else:
        out['loss'] = out['pg_loss'] + kl_coef * out['kl_loss']
    return out
