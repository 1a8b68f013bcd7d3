"""Generate the NewFC training goldens (tests/golden/newfc_train_small.npz, newfc_scst_full.npz) from the LIVE reference.

    python tests/make_newfc_golden.py [small] [full]      # needs the reference checkout that oracle/make_golden.py reads

The reference's NewFCModel runs as published, in train mode with every dropout probability set to 0, and gets the region features the
reference loader hands a NewFC model: att_feats of shape [B, 0, 0] and att_masks None (opts.py if_use_feat, dataloader.py:232-241,284).
Weights and inputs come from the seeded generators (synthetic.make_weights('newfc', ...), make_inputs), so the tests rebuild them from the
stored seeds.

* small (B = 4, small dimensions), all 9 parameter gradients stored in full:
  'xe'  LanguageModelCriterion of the teacher-forced _forward over labels[..., :-1] (seq_per_img 3);
  'ls'  LabelSmoothing(0.2) of the same forward;
  'rl'  RewardCriterion of the reference's own multinomial draw (sample_n 3, stored) with a fixed per-row reward.
* full (configs/fc_rl.yml / fc_nsc.yml sizes: E = H = 512, F_fc = 2048, V = 9487, T = 20, 10 images x 5 samples): the references are
  corrupted copies of the model's greedy captions, scored by the reference's own CIDEr-D scorer;
  'sc'  LossWrapper(sc_flag=True) + backward();
  'nsc' LossWrapper(struc_flag=True) with structure_loss_type 'new_self_critical', weight 1, + backward().
  The samples are stored (the engine replays them as forced tokens) and every gradient as a _subsample fingerprint.
"""
from __future__ import annotations

import argparse
import json
import os
import pickle
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
sys.path.insert(0, REPO)
sys.path.insert(0, HERE)

from oracle import caption_oracle as co                                       # noqa: E402
from oracle import ciderd_oracle as cdo                                       # noqa: E402
from oracle.make_golden import _enter_scratch, _subsample, ref_model          # noqa: E402

SMALL = dict(V=60, E=32, H=32, A=16, F_fc=48, F_att=48, T=8)
SEED, LOGIT_SCALE, B = 23, 20.0, 4
FULL = dict(V=9487, E=512, H=512, A=512, F_fc=2048, F_att=2048, T=20)
FULL_B, FULL_N, FULL_SEED, FULL_LOGIT_SCALE = 10, 5, 1234, 12.0


def labels_for(seed, N, T, V):
    g = torch.Generator().manual_seed(seed)
    labels = torch.zeros(N, T + 2, dtype=torch.long)
    for i in range(N):
        L = int(torch.randint(2, T + 1, (1,), generator=g))
        labels[i, 1:1 + L] = torch.randint(1, V + 1, (L,), generator=g)
    masks = torch.zeros(N, T + 2)
    for i in range(N):
        masks[i, :int((labels[i, 1:] > 0).sum()) + 2] = 1
    return labels, masks


def no_dropout(m):
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
    m.train()


def gen_small(out_dir):
    from captioning.modules.losses import LabelSmoothing, LanguageModelCriterion, RewardCriterion
    W = co.make_weights('newfc', SMALL['V'], SMALL['E'], SMALL['H'], SMALL['A'], SMALL['F_fc'], SMALL['F_att'], seed=SEED, logit_scale=LOGIT_SCALE)
    fc, _ = co.make_inputs(B, 1, SMALL['F_fc'], SMALL['F_att'], seed=SEED)
    att = fc.new_zeros(B, 0, 0)
    T, V = SMALL['T'], SMALL['V']
    m = ref_model('newfc', W=W, **SMALL)
    no_dropout(m)
    names = [k for k, _ in m.named_parameters()]
    res = {}
    labels, lmasks = labels_for(7, B * 3, T, V)
    res['xe_labels'], res['xe_masks'] = labels.numpy(), lmasks.numpy()
    for tag, crit in (('xe', LanguageModelCriterion()), ('ls', LabelSmoothing(smoothing=0.2))):
        m.zero_grad()
        lp = m(fc, att, labels[:, :-1].reshape(B, 3, -1), None, mode='forward')
        loss = crit(lp, labels[:, 1:], lmasks[:, 1:])
        loss.backward()
        res[tag + '_loss'] = np.array(float(loss))
        for k, p in m.named_parameters():
            res[tag + '_grad_' + k] = p.grad.numpy().copy()
    m.zero_grad()
    n = 3
    torch.manual_seed(9)
    seq, lp = m(fc, att, None, opt={'sample_method': 'sample', 'beam_size': 1, 'sample_n': n}, mode='sample')
    reward = torch.linspace(-1.0, 1.5, B * n).unsqueeze(1).expand(B * n, T).contiguous()
    loss = RewardCriterion()(lp, seq, reward)
    loss.backward()
    res['rl_seq'], res['rl_reward'], res['rl_loss'], res['rl_lp'] = seq.numpy(), reward.numpy(), np.array(float(loss)), lp.detach().numpy()
    for k, p in m.named_parameters():
        res['rl_grad_' + k] = p.grad.numpy().copy()
    meta = {'seed': SEED, 'logit_scale': LOGIT_SCALE, 'B': B, 'params': names}
    np.savez_compressed(os.path.join(out_dir, 'newfc_train_small.npz'), cfg=np.array([SMALL[k] for k in ('V', 'E', 'H', 'A', 'F_fc', 'F_att', 'T')]),
                        meta=np.array(json.dumps(meta)), **res)
    print('newfc_train_small: xe loss %.5f, ls loss %.5f, rl loss %.5f, rl lengths %s' %
          (res['xe_loss'], res['ls_loss'], res['rl_loss'], (res['rl_seq'] > 0).sum(1).tolist()))


def gen_full(out_dir, scratch):
    from captioning.modules.loss_wrapper import LossWrapper
    from captioning.utils import rewards as R
    cfg = FULL
    Bf, n = FULL_B, FULL_N
    W = co.make_weights('newfc', cfg['V'], cfg['E'], cfg['H'], cfg['A'], cfg['F_fc'], cfg['F_att'], seed=FULL_SEED, logit_scale=FULL_LOGIT_SCALE)
    fc, _ = co.make_inputs(Bf, 1, cfg['F_fc'], cfg['F_att'], seed=FULL_SEED)
    att = fc.new_zeros(Bf, 0, 0)
    m = ref_model('newfc', W=W, **cfg)
    no_dropout(m)
    # references: corrupted copies of each image's greedy caption (as gen_aoa_scst_full) so CIDEr-D gives O(1) scores and spread rewards
    m.eval()
    with torch.no_grad():
        g0, _ = m(fc, att, None, opt={'sample_method': 'greedy', 'beam_size': 1}, mode='sample')
    m.train()
    rng = np.random.RandomState(5)
    gts = []
    for i in range(Bf):
        rows = np.zeros((5, 16), np.int64)
        for j in range(5):
            ln = 16 if j < 2 else int(rng.randint(6, 15))
            row = g0[i, :ln].numpy().copy()
            flip = rng.rand(ln) < 0.3
            row[flip] = rng.randint(1, cfg['V'] + 1, size=int(flip.sum()))
            rows[j, :ln] = row
        gts.append(rows)
    df, ref_len = cdo.build_document_frequency(cdo.make_refs(1000, cfg['V'], seed=4) + gts)
    from collections import defaultdict
    dd = defaultdict(float)
    dd.update({tuple(str(t) for t in k): v for k, v in df.items()})
    with open(os.path.join(scratch, 'data', 'newfc-full-df.p'), 'wb') as f:
        pickle.dump({'document_frequency': dd, 'ref_len': ref_len}, f, protocol=2)
    R.CiderD_scorer = None
    R.Cider_scorer = None
    R.init_scorer('newfc-full-df')
    res = {'gts': np.stack(gts).astype(np.int16)}
    names = [k for k, _ in m.named_parameters()]
    for tag, sc_flag, struc_flag in (('sc', True, False), ('nsc', False, True)):
        opt = argparse.Namespace(label_smoothing=0, structure_loss_type='new_self_critical', structure_loss_weight=1, train_sample_method='sample',
                                 train_beam_size=1, train_sample_n=n, sc_sample_method='greedy', sc_beam_size=1, cider_reward_weight=1.0,
                                 bleu_reward_weight=0.0, use_ppo=0, struc_use_logsoftmax=1, entropy_reward_weight=0, self_cider_reward_weight=0)
        lw = LossWrapper(m, opt)
        captured = []
        orig = m._sample

        def spy(*a, **k):
            out = orig(*a, **k)
            captured.append(out[0].detach().clone())
            return out
        m._sample = spy
        torch.manual_seed(77 if tag == 'sc' else 78)
        m.zero_grad()
        out = lw(fc, att, None, None, None, gts, torch.arange(Bf), sc_flag, struc_flag, False)
        out['loss'].backward()
        m._sample = orig
        sample_seq = captured[-1]
        assert sample_seq.shape == (Bf * n, cfg['T'])
        res[tag + '_sample_seq'] = sample_seq.numpy().astype(np.int16)
        res[tag + '_loss'] = out['loss'].detach().numpy()
        if tag == 'sc':
            greedy_seq = captured[0]
            reward = R.get_self_critical_reward(greedy_seq, gts, sample_seq, opt)
            res['sc_greedy_seq'] = greedy_seq.numpy().astype(np.int16)
            res['sc_reward'] = reward[:, 0].astype(np.float64)
        else:
            res['nsc_scores'] = out['reward'].detach().numpy().astype(np.float64).reshape(-1)
        for k, prm in m.named_parameters():
            sub, step, stats = _subsample(prm.grad)
            res['%s_g_%s' % (tag, k)], res['%s_s_%s' % (tag, k)], res['%s_t_%s' % (tag, k)] = sub, step, stats
        print('newfc_scst_full %s: loss %.6g, sample lengths %s' % (tag, float(out['loss']), (sample_seq > 0).sum(1)[:10].tolist()))
    keys = np.array([list(k) + [-1] * (4 - len(k)) for k in df.keys()], np.int32)
    vals = np.array(list(df.values()), np.float64)
    np.savez_compressed(os.path.join(out_dir, 'newfc_scst_full.npz'), cfg=np.array([cfg[k] for k in ('V', 'E', 'H', 'A', 'F_fc', 'F_att', 'T')]),
                        meta=np.array([Bf, n, FULL_SEED]), logit_scale=np.array(FULL_LOGIT_SCALE), df_keys=keys, df_vals=vals, ref_len=np.array(ref_len),
                        names=np.array(names), **res)


def main():
    out_dir = os.path.join(REPO, 'tests', 'golden')
    scratch = _enter_scratch()
    torch.set_num_threads(os.cpu_count())
    which = sys.argv[1:] or ['small', 'full']
    if 'small' in which:
        gen_small(out_dir)
    if 'full' in which:
        gen_full(out_dir, scratch)


if __name__ == '__main__':
    main()
