"""Generate the Att2in2 goldens (tests/golden/att2in2_small.npz, att2in2_b32.npz, att2in2_state_dict_keys.json) from the LIVE reference.

    python tests/make_att2in2_golden.py [small] [b32] [keys]      # needs the reference checkout that oracle/make_golden.py reads

The reference's Att2in2Model runs as published for every case except diverse beam search, which needs the one-line repair of
tests/make_dbs_golden.py (add_diversity calls a repeat_tensor method that does not exist).  Weights and inputs come from the seeded
generators (synthetic.make_weights('att2in2', ...), make_inputs), so the tests rebuild the same inputs from the stored seeds.

Training cases run the reference model in train mode with drop_prob_lm = 0 and back-propagate:
* 'xe': LanguageModelCriterion of the teacher-forced _forward over labels[..., :-1] against labels[..., 1:];
* 'rl': RewardCriterion of the reference's own multinomial draw (sample_n rows per image, stored) with a fixed per-row reward, the loss
  the SCST step and the 'new_self_critical' structure loss apply to the engine's samples.
Every one of the 17 parameter gradients is stored in full.
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
import att2in2_oracle as ao                                      # noqa: E402
import dbs_oracle                                                # noqa: E402
from make_dbs_golden import install_shim, run_case               # noqa: E402

SMALL = dict(V=60, E=32, H=32, A=16, F_fc=48, F_att=48, T=8)
SEED, LOGIT_SCALE, B, R = 21, 20.0, 4, 7


def small_masks():
    masks = torch.ones(B, R)
    masks[1, 5:] = 0
    masks[3, 3:] = 0
    return masks


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


def gen_small(out_dir):
    from captioning.modules.losses import LanguageModelCriterion, RewardCriterion
    W = co.make_weights('att2in2', SMALL['V'], SMALL['E'], SMALL['H'], SMALL['A'], SMALL['F_fc'], SMALL['F_att'], seed=SEED, logit_scale=LOGIT_SCALE)
    fc, att = co.make_inputs(B, R, SMALL['F_fc'], SMALL['F_att'], seed=SEED)
    masks = small_masks()
    T, V = SMALL['T'], SMALL['V']
    m = ref_model('att2in2', W=W, **SMALL)
    res = {}
    with torch.no_grad():
        for tag, mk in (('', None), ('masked_', masks)):
            seq, lp = m(fc, att, mk, opt={'sample_method': 'greedy', 'beam_size': 1}, mode='sample')
            res[tag + 'greedy_seq'], res[tag + 'greedy_lp'] = seq.numpy(), lp.numpy()
        torch.manual_seed(5)
        seq, lp = m(fc, att, None, opt={'sample_method': 'sample', 'beam_size': 1, 'sample_n': 3, 'temperature': 1.0}, mode='sample')
        res['sample_seq'], res['sample_lp'] = seq.numpy(), lp.numpy()
        labels, lmasks = labels_for(3, B * 2, T, V)
        res['tf_labels'], res['tf_lp'] = labels.numpy(), m(fc, att, labels[:, :-1].reshape(B, 2, -1), None, mode='forward').numpy()
        for name, beam, G, lam, extra, mk in (('beam_wu', 4, 1, 0.0, {'length_penalty': 'wu_0.5'}, None),
                                             ('beam_constraint', 4, 1, 0.0, {'decoding_constraint': 1}, None),
                                             ('beam_masked', 4, 1, 0.0, {}, masks),
                                             ('dbs', 6, 3, 0.5, {}, None)):
            out = run_case(m, fc, att, mk, beam, G, lam, extra, T)
            for k, v in out.items():
                res['%s_%s' % (name, k)] = v
    # training: train mode, dropout 0 (drop_prob_lm is a module attribute of the Dropout layers)
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
    m.train()
    names = [k for k, _ in m.named_parameters()]
    m.zero_grad()
    labels, lmasks = labels_for(7, B * 3, T, V)
    lp = m(fc, att, labels[:, :-1].reshape(B, 3, -1), masks, mode='forward')
    loss = LanguageModelCriterion()(lp, labels[:, 1:], lmasks[:, 1:])
    loss.backward()
    res['xe_labels'], res['xe_masks'], res['xe_loss'] = labels.numpy(), lmasks.numpy(), np.array(float(loss))
    for k, p in m.named_parameters():
        res['xe_grad_' + k] = p.grad.numpy().copy()
    m.zero_grad()
    n = 3
    torch.manual_seed(9)
    seq, lp = m(fc, att, masks, opt={'sample_method': 'sample', 'beam_size': 1, 'sample_n': n}, mode='sample')
    reward = torch.linspace(-1.0, 1.5, B * n).unsqueeze(1).expand(B * n, T).contiguous()
    loss = RewardCriterion()(lp, seq, reward)
    loss.backward()
    res['rl_seq'], res['rl_reward'], res['rl_loss'] = seq.numpy(), reward.numpy(), np.array(float(loss))
    for k, p in m.named_parameters():
        res['rl_grad_' + k] = p.grad.numpy().copy()
    meta = {'seed': SEED, 'logit_scale': LOGIT_SCALE, 'B': B, 'R': R, 'params': names}
    np.savez_compressed(os.path.join(out_dir, 'att2in2_small.npz'), cfg=np.array([SMALL[k] for k in ('V', 'E', 'H', 'A', 'F_fc', 'F_att', 'T')]),
                        meta=np.array(json.dumps(meta)), **res)
    print('att2in2_small: greedy[0]', res['greedy_seq'][0].tolist(), 'xe loss %.4f rl loss %.4f' % (res['xe_loss'], res['rl_loss']))


def gen_b32(out_dir):
    """a2i2 recipe size (E = H = A = 512, V = 9487, T = 20), batch 32, beam 5, with each image's smallest candidate gap from the restatement
    so the GPU test can demand bit-exact ids wherever a decision is not a near tie."""
    cfg = dict(V=9487, E=512, H=512, A=512, F_fc=2048, F_att=2048, T=20)
    Bb, Rb, beam, seed = 32, 36, 5, 1234
    W = co.make_weights('att2in2', cfg['V'], cfg['E'], cfg['H'], cfg['A'], cfg['F_fc'], cfg['F_att'], seed=seed, logit_scale=12.0)
    fc, att = co.make_inputs(Bb, Rb, cfg['F_fc'], cfg['F_att'], seed=seed)
    m = ref_model('att2in2', W=W, **cfg)
    with torch.no_grad():
        out = run_case(m, fc, att, None, beam, 1, 0.0, {}, cfg['T'])
        rows = []
        _, _, odone = co.sample_beam(ao.Att2in2Family(W, cfg['T']), fc, att, beam_size=beam, margin_rows=rows)
    margin = torch.stack(rows, 1).min(1).values.numpy()
    oseqs, _, _ = dbs_oracle.beams_to_arrays(odone, beam, cfg['T'])
    agree = (oseqs == out['done_seq']).all((1, 2))
    np.savez_compressed(os.path.join(out_dir, 'att2in2_b32.npz'), cfg=np.array([cfg[k] for k in ('V', 'E', 'H', 'A', 'F_fc', 'F_att', 'T')]),
                        meta=np.array([Bb, Rb, beam, seed]), seq=out['seq'].astype(np.int16), picked=out['picked'],
                        done_seq=out['done_seq'].astype(np.int16), done_len=out['done_len'].astype(np.int8), done_p=out['done_p'], image_margin=margin)
    print('att2in2_b32: restatement agrees with the reference on %d / %d images; smallest margin %.3g' % (int(agree.sum()), Bb, float(margin.min())))


def gen_keys(out_dir):
    cfg = dict(V=60, E=32, H=40, A=16, F_fc=48, F_att=56, T=8)
    W = co.make_weights('att2in2', cfg['V'], cfg['E'], cfg['H'], cfg['A'], cfg['F_fc'], cfg['F_att'], seed=1)
    m = ref_model('att2in2', W=W, **cfg)
    keys = {k: list(v.shape) for k, v in m.state_dict().items()}
    json.dump({'cfg': cfg, 'keys': keys}, open(os.path.join(out_dir, 'att2in2_state_dict_keys.json'), 'w'), indent=1)


def main():
    out_dir = os.path.join(REPO, 'tests', 'golden')
    _enter_scratch()
    install_shim()
    torch.set_num_threads(os.cpu_count())
    which = sys.argv[1:] or ['small', 'b32', 'keys']
    if 'keys' in which:
        gen_keys(out_dir)
    if 'small' in which:
        gen_small(out_dir)
    if 'b32' in which:
        gen_b32(out_dir)


if __name__ == '__main__':
    main()
