"""Generate tests/golden/logit_layers_small.npz from the LIVE reference: UpDown, Att2in2, NewFC and AoANet with logit_layers = 3.

    python tests/make_logit_layers_golden.py          # needs the reference checkout that oracle/make_golden.py reads

With logit_layers = k > 1 AttModel replaces its vocabulary Linear by k - 1 hidden [Linear(H, H), ReLU, Dropout(0.5)] blocks ahead of it
(AttModel.py:87-92; AoAModel inherits it).  The reference runs as published but for one repair: AttModel.py calls ``reduce`` there
without importing it (a Python 2 builtin, functools.reduce under Python 3), so the script puts functools.reduce into that module's namespace
before building the models.  Weights and inputs come from the seeded generators (synthetic.make_weights(..., logit_layers=3),
make_inputs) and are loaded into the reference's own modules with load_state_dict(strict=True).  Per family (prefix '<family>_'):
* 'keys': the state_dict's names and shapes (in meta);
* greedy ids and log-probs; beam search with beam 3 (seq and done_beams' seq / logps / p); teacher-forced log-probs;
* the XE loss (LanguageModelCriterion of the teacher-forced _forward over labels[..., :-1] against labels[..., 1:]) and every parameter
  gradient, in eval mode, so that no dropout draw is involved.
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
from oracle.make_golden import _enter_scratch, beams_to_arrays, ref_model     # noqa: E402

K = 3
CFG = dict(V=60, E=32, H=32, A=16, F_fc=48, F_att=48, T=8)
SEED, LOGIT_SCALE, B, R, BEAM = 31, 20.0, 4, 7, 3
FAMILIES = ('updown', 'att2in2', 'newfc', 'aoa')
AOA = dict(num_layers=2, refine=1, refine_aoa=1, use_ff=0, decoder_type='AoA', use_multi_head=2, num_heads=4, multi_head_scale=1, mean_feats=1,
           ctx_drop=1, dropout_aoa=0.3)


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


def gen(out_dir):
    import functools
    import captioning.models        # noqa: F401  (its package namespace re-exports the class AttModel under the module's name)
    from captioning.modules.losses import LanguageModelCriterion
    sys.modules['captioning.models.AttModel'].reduce = functools.reduce
    fc, att = co.make_inputs(B, R, CFG['F_fc'], CFG['F_att'], seed=SEED)
    T, V = CFG['T'], CFG['V']
    res, keys = {}, {}
    for fam in FAMILIES:
        W = co.make_weights(fam, CFG['V'], CFG['E'], CFG['H'], CFG['A'], CFG['F_fc'], CFG['F_att'], seed=SEED, logit_scale=LOGIT_SCALE,
                            logit_layers=K)
        m = ref_model(fam, W=W, logit_layers=K, **CFG, **(AOA if fam == 'aoa' else {}))
        keys[fam] = {k: list(v.shape) for k, v in m.state_dict().items()}
        p = fam + '_'
        with torch.no_grad():
            seq, lp = m(fc, att, None, opt={'sample_method': 'greedy', 'beam_size': 1}, mode='sample')
            res[p + 'greedy_seq'], res[p + 'greedy_lp'] = seq.numpy(), lp.numpy()
            seq, _ = m(fc, att, None, opt={'beam_size': BEAM, 'sample_n': 1}, mode='sample')
            res[p + 'beam_seq'] = seq.numpy()
            dseq, dlen, dp = beams_to_arrays(m.done_beams, BEAM, T)
            logps = np.zeros((B, BEAM, T, V + 1), np.float32)
            for i, lst in enumerate(m.done_beams):
                for j, rec in enumerate(lst):
                    logps[i, j, :rec['logps'].shape[0]] = rec['logps'].numpy()
            res[p + 'beam_done_seq'], res[p + 'beam_done_p'], res[p + 'beam_done_logps'] = dseq, dp, logps
        labels, lmasks = labels_for(3, B * 2, T, V)
        m.zero_grad()
        with torch.enable_grad():
            lp = m(fc, att, labels[:, :-1], None, mode='forward')
            loss = LanguageModelCriterion()(lp, labels[:, 1:], lmasks[:, 1:])
            loss.backward()
        res[p + 'tf_lp'] = lp.detach().numpy()
        res[p + 'xe_loss'] = np.array(float(loss))
        for name, prm in m.named_parameters():
            res[p + 'grad_' + name] = prm.grad.numpy().copy() if prm.grad is not None else np.zeros(tuple(prm.shape), np.float32)
        res[p + 'tf_labels'], res[p + 'tf_masks'] = labels.numpy(), lmasks.numpy()
        print('%s: k = %d, %d tensors, greedy lengths %s, xe loss %.5f' % (fam, K, len(keys[fam]), (seq > 0).sum(1).tolist(), float(loss)))
    meta = dict(seed=SEED, logit_scale=LOGIT_SCALE, B=B, R=R, beam=BEAM, logit_layers=K, keys=keys)
    np.savez_compressed(os.path.join(out_dir, 'logit_layers_small.npz'), cfg=np.array([CFG[k] for k in ('V', 'E', 'H', 'A', 'F_fc', 'F_att', 'T')]),
                        meta=json.dumps(meta), **res)


if __name__ == '__main__':
    out_dir = os.path.join(HERE, 'golden')
    torch.set_grad_enabled(False)
    _enter_scratch()
    gen(out_dir)
