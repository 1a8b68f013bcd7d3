"""Generate the diverse beam search goldens (tests/golden/dbs_small.npz, tests/golden/updown_dbs_b32.npz) from the LIVE reference.

    python tests/make_dbs_golden.py [small] [b32]        # needs the reference checkout that oracle/make_golden.py reads

The reference cannot run diverse beam search as published: add_diversity calls ``self.repeat_tensor(bdash, change)``
(captioning/models/CaptionModel.py:53), which no class defines, and raises AttributeError at the first step of group 1 past its first
position.  This script applies exactly one shim before running it,

    CaptionModel.repeat_tensor = lambda self, n, x: repeat_tensors(n, x)

with repeat_tensors from captioning/models/utils.py, the function the call was meant to reach.  Nothing else in the reference is changed.
Weights and inputs come from the seeded oracle.caption_oracle generators, so the tests regenerate the same inputs from the stored seeds.
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
sys.path.insert(0, REPO)
sys.path.insert(0, HERE)

from oracle import caption_oracle as co                         # noqa: E402
from oracle.make_golden import _enter_scratch, ref_model         # noqa: E402
import dbs_oracle                                                # noqa: E402

SMALL = dict(V=60, E=32, H=32, A=16, F_fc=48, F_att=48, T=8)
AOA_EXTRA = dict(num_layers=2, refine=1, refine_aoa=1, use_ff=0, decoder_type='AoA', use_multi_head=2, num_heads=4, multi_head_scale=1, mean_feats=1,
                 ctx_drop=1, dropout_aoa=0.3)
# (name, beam_size, group_size, diversity_lambda, extra options, masked)
CASES = [('b4g2_l05', 4, 2, 0.5, {}, False), ('b4g2_l2', 4, 2, 2.0, {}, False),
         ('b6g3_l05', 6, 3, 0.5, {}, False), ('b6g3_l2', 6, 3, 2.0, {}, False),
         ('b4g4_l05', 4, 4, 0.5, {}, False), ('b4g4_l2', 4, 4, 2.0, {}, False),
         ('wu', 6, 3, 0.5, {'length_penalty': 'wu_0.5'}, False),
         ('constraint', 6, 3, 0.5, {'decoding_constraint': 1}, False),
         ('temp', 4, 2, 0.5, {'temperature': 1.3}, False),
         ('masked', 6, 3, 0.5, {}, True),
         ('samplen', 6, 3, 0.5, {'sample_n': 2}, False)]


def install_shim():
    from captioning.models.CaptionModel import CaptionModel
    from captioning.models.utils import repeat_tensors
    CaptionModel.repeat_tensor = lambda self, n, x: repeat_tensors(n, x)


def case_masks(B, R):
    masks = torch.ones(B, R)
    masks[1, 5:] = 0
    masks[3, 3:] = 0
    return masks


def run_case(m, fc, att, masks, beam, G, lam, extra, T):
    opt = dict({'beam_size': beam, 'group_size': G, 'diversity_lambda': lam, 'sample_n': 1}, **extra)
    seq, lp = m(fc, att, masks, opt=opt, mode='sample')
    picked = lp.gather(2, seq.unsqueeze(2)).squeeze(2)
    dseq, dlen, dp = dbs_oracle.beams_to_arrays(m.done_beams, beam, T)
    V1 = lp.shape[2]
    logps = np.zeros((beam, T, V1), np.float32)           # the full rows of image 0's records
    for j, rec in enumerate(m.done_beams[0]):
        logps[j, :rec['logps'].shape[0]] = rec['logps'].numpy()
    return {'seq': seq.numpy(), 'picked': picked.numpy(), 'done_seq': dseq, 'done_len': dlen, 'done_p': dp, 'logps0': logps}


def gen_small(out_dir):
    res, meta = {}, {}
    B, R = 4, 7
    for family, seed, extra in (('updown', 11, {}), ('aoa', 17, AOA_EXTRA)):
        W = co.make_weights(family, SMALL['V'], SMALL['E'], SMALL['H'], SMALL['A'], SMALL['F_fc'], SMALL['F_att'], seed=seed, logit_scale=20.0)
        fc, att = co.make_inputs(B, R, SMALL['F_fc'], SMALL['F_att'], seed=seed)
        m = ref_model(family, W=W, **SMALL, **extra)
        meta[family] = {'seed': seed, 'logit_scale': 20.0, 'B': B, 'R': R}
        with torch.no_grad():
            for name, beam, G, lam, opts, masked in CASES:
                out = run_case(m, fc, att, case_masks(B, R) if masked else None, beam, G, lam, opts, SMALL['T'])
                for k, v in out.items():
                    res['%s_%s_%s' % (family, name, k)] = v
                print(family, name, 'seq[0]', out['seq'][0].tolist(), 'p', np.round(out['done_p'][0], 3).tolist())
    cases = [{'name': n, 'beam_size': b, 'group_size': g, 'diversity_lambda': l, 'opts': o, 'masked': mk} for n, b, g, l, o, mk in CASES]
    np.savez_compressed(os.path.join(out_dir, 'dbs_small.npz'), cfg=np.array([SMALL[k] for k in ('V', 'E', 'H', 'A', 'F_fc', 'F_att', 'T')]),
                        cases=np.array(json.dumps(cases)), meta=np.array(json.dumps(meta)), **res)


def gen_b32(out_dir):
    """UpDown at BASELINE.json configs[1] dimensions, batch 32, beam 9 in 3 groups.  Also stores each image's smallest candidate gap over all
    group steps (from the restatement on the same inputs), so the GPU test can demand bit-exact ids wherever the decision is not a tie."""
    cfg = dict(V=9487, E=1000, H=1000, A=512, F_fc=2048, F_att=2048, T=20)
    B, R, beam, G, lam, seed = 32, 36, 9, 3, 0.5, 1234
    W = co.make_weights('updown', cfg['V'], cfg['E'], cfg['H'], cfg['A'], cfg['F_fc'], cfg['F_att'], seed=seed, logit_scale=12.0)
    fc, att = co.make_inputs(B, R, cfg['F_fc'], cfg['F_att'], seed=seed)
    m = ref_model('updown', W=W, **cfg)
    with torch.no_grad():
        out = run_case(m, fc, att, None, beam, G, lam, {}, cfg['T'])
        rows = []
        oseq, _, odone = dbs_oracle.diverse_sample_beam(co.Family('updown', W, cfg['T']), fc, att, beam_size=beam, group_size=G, diversity_lambda=lam,
                                                        margin_rows=rows)
    margin = torch.stack(rows, 1).min(1).values.numpy()
    oseqs, _, _ = dbs_oracle.beams_to_arrays(odone, beam, cfg['T'])
    agree = (oseqs == out['done_seq']).all((1, 2))
    np.savez_compressed(os.path.join(out_dir, 'updown_dbs_b32.npz'), cfg=np.array([cfg[k] for k in ('V', 'E', 'H', 'A', 'F_fc', 'F_att', 'T')]),
                        meta=np.array([B, R, beam, G, seed]), diversity_lambda=np.array(lam), seq=out['seq'].astype(np.int16), picked=out['picked'],
                        done_seq=out['done_seq'].astype(np.int16), done_len=out['done_len'].astype(np.int8), done_p=out['done_p'], image_margin=margin)
    print('updown_dbs_b32: restatement agrees with the reference on %d / %d images; smallest margin %.3g; %d images below 1e-3' %
          (int(agree.sum()), B, float(margin.min()), int((margin < 1e-3).sum())))


def main():
    out_dir = os.path.join(REPO, 'tests', 'golden')
    os.makedirs(out_dir, exist_ok=True)
    _enter_scratch()
    install_shim()
    torch.set_num_threads(os.cpu_count())
    which = sys.argv[1:] or ['small', 'b32']
    if 'small' in which:
        gen_small(out_dir)
    if 'b32' in which:
        gen_b32(out_dir)


if __name__ == '__main__':
    main()
