"""Generate the PPO golden (tests/golden/ppo_small.npz) from the LIVE reference's PPOLoss (losses.py:267-357).

    python tests/make_ppo_golden.py      # needs the reference checkout that oracle/make_golden.py reads

A small UpDown model holds the old policy's weights (synthetic.make_weights, seed OLD_SEED); its state dict is saved to a scratch file and
PPOLoss(opt, model) builds the old policy the reference's way -- copy.deepcopy of the model, torch.load + load_state_dict of that file, eval
mode, no gradients.  The sampled side is fixed data: captions `seq` (some finished early), log-probs `lp` = log_softmax of the old policy's
own teacher-forced rows plus noise (rows after a caption's end zeroed, as _sample leaves them), and the scores get_scores would return
(patched in).  The noise puts some policy ratios inside [1 - eps, 1 + eps] and some outside.  Both reductions are stored with
loss.backward() gradients with respect to lp ('mean': of the loss; 'none': of the sum of the row losses).
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
sys.path.insert(0, REPO)
sys.path.insert(0, HERE)

from oracle import caption_oracle as co                     # noqa: E402
from oracle.make_golden import _enter_scratch, ref_model    # noqa: E402

SMALL = dict(V=30, E=16, H=16, A=8, F_fc=12, F_att=12, T=7)
B, N_PER, R = 3, 4, 5
OLD_SEED, LOGIT_SCALE, DATA_SEED = 17, 4.0, 3
CLIPRANGE, KL_COEF = 0.2, 0.02


def captions(N, T, V, g):
    seq = torch.zeros(N, T, dtype=torch.long)
    for i in range(N):
        L = int(torch.randint(1, T + 1, (1,), generator=g))         # L = T: no EOS inside the window
        seq[i, :L] = torch.randint(1, V + 1, (L,), generator=g)
    return seq


def main(out_dir):
    scratch = _enter_scratch()
    from captioning.modules import losses
    W = co.make_weights('updown', *(SMALL[k] for k in ('V', 'E', 'H', 'A', 'F_fc', 'F_att')), seed=OLD_SEED, logit_scale=LOGIT_SCALE)
    fc, att = co.make_inputs(B, R, SMALL['F_fc'], SMALL['F_att'], seed=DATA_SEED)
    T, V, N = SMALL['T'], SMALL['V'], B * N_PER
    g = torch.Generator().manual_seed(DATA_SEED)
    seq = captions(N, T, V, g)
    scores = torch.rand(N, generator=g, dtype=torch.float64) * 2.0
    path = os.path.join(scratch, 'old_model.pth')
    torch.save(W, path)

    # the policy being trained: the same architecture with other weights; PPOLoss copies it and loads the old weights into the copy
    model = ref_model('updown', W=co.make_weights('updown', *(SMALL[k] for k in ('V', 'E', 'H', 'A', 'F_fc', 'F_att')), seed=OLD_SEED + 1,
                                                  logit_scale=LOGIT_SCALE), **SMALL)
    opt = argparse.Namespace(use_ppo=1, ppo_old_model_path=path, ppo_cliprange=CLIPRANGE, ppo_kl_coef=KL_COEF, train_sample_n=N_PER)
    crit = losses.PPOLoss(opt, model)
    losses.get_scores = lambda data_gts, seq_, opt_: scores.numpy()
    gts = [np.zeros((1, T), np.int64) for _ in range(B)]

    with torch.no_grad():
        lo = crit.old_model(fc, att, torch.cat([seq.new_zeros(N, 1), seq[:, :-1]], 1), None)
    live = torch.cat([torch.ones(N, 1), (seq[:, :-1] > 0).float()], 1)
    lp0 = torch.log_softmax(lo + 0.25 * torch.randn(lo.shape, generator=g), dim=2) * live.unsqueeze(2)

    res = {'cfg': np.array([SMALL[k] for k in ('V', 'E', 'H', 'A', 'F_fc', 'F_att', 'T')]), 'dims': np.array([B, N_PER, R]),
           'hyper': np.array([CLIPRANGE, KL_COEF]), 'fc': fc.numpy(), 'att': att.numpy(), 'seq': seq.numpy(), 'scores': scores.numpy(),
           'lp': lp0.numpy(), 'lo': lo.numpy()}
    for k, v in W.items():
        res['w:' + k] = v.numpy()
    for reduction in ('mean', 'none'):
        lp = lp0.clone().requires_grad_(True)
        out = crit(lp, seq, gts, fc, att, None, reduction=reduction)
        (out['loss'] if reduction == 'mean' else out['loss'].sum()).backward()
        for k in ('loss', 'pg_loss', 'kl_loss', 'clipfrac', 'reward'):
            res['%s_%s' % (reduction, k)] = out[k].detach().numpy()
        res['%s_dlp' % reduction] = lp.grad.numpy()
    ratio = np.exp(np.take_along_axis(lp0.numpy(), seq.numpy()[..., None], 2) - np.take_along_axis(lo.numpy(), seq.numpy()[..., None], 2))[..., 0]
    m = live.numpy() > 0
    print('clipped %d of %d live positions' % (int((np.abs(ratio[m] - 1) > CLIPRANGE).sum()), int(m.sum())))
    np.savez_compressed(os.path.join(out_dir, 'ppo_small.npz'), **res)


if __name__ == '__main__':
    main(os.path.join(HERE, 'golden'))
