"""Generate the test-time ensemble golden (tests/golden/ensemble_small.npz) from the LIVE reference's AttEnsemble.

    python tests/make_ensemble_golden.py          # needs the reference checkout that oracle/make_golden.py reads

AttEnsemble (captioning/models/AttEnsemble.py) calls CaptionModel.__init__ but not AttModel.__init__, so the published class has no
bos_idx / eos_idx / pad_idx / unk_idx / vocab, which AttModel._sample, _sample_beam and CaptionModel.beam_search read: every decode raises
AttributeError as published.  This script applies exactly one shim after constructing it,

    ens.bos_idx, ens.eos_idx, ens.pad_idx, ens.unk_idx, ens.vocab = (the same attributes of models[0])

-- the values AttModel.__init__ would have set, taken from models[0] as AttEnsemble takes vocab_size / seq_length.  Nothing else in the
reference is changed.  Members are reference models loaded with the seeded synthetic weights of oracle.caption_oracle.make_weights, so the
tests rebuild the same members and inputs from the stored seeds.
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
from oracle.make_golden import _enter_scratch, beams_to_arrays, ref_model   # noqa: E402
import ensemble_oracle as eo                                    # noqa: E402

SMALL = dict(V=60, E=32, H=32, A=16, F_fc=48, F_att=48, T=8)
AOA_EXTRA = dict(num_layers=2, refine=1, refine_aoa=1, use_ff=0, decoder_type='AoA', use_multi_head=2, num_heads=4, multi_head_scale=1, mean_feats=1,
                 ctx_drop=1, dropout_aoa=0.3)
AOA_HEADS = 4
LOGIT_SCALE = 10.0
B, R, INPUT_SEED, LABEL_SEED = 4, 7, 23, 29
# mix name -> [(family, weight seed)]; weight sets: equal (None) and unequal
MIXES = {'updown2': [('updown', 11), ('updown', 12)],
         'mixed3': [('updown', 11), ('att2in2', 13), ('aoa', 17)],
         'newfc_updown': [('newfc', 3), ('updown', 12)]}
WEIGHTS = {'eq': None, 'uneq': {2: [1.0, 2.0], 3: [1.0, 2.0, 0.5]}}
# (name, options of forward(..., mode='sample') or 'teacher', masked)
CASES = [('greedy', {'sample_method': 'greedy', 'beam_size': 1}, False),
         ('beam3', {'beam_size': 3, 'sample_n': 1}, True),
         ('beam5', {'beam_size': 5, 'sample_n': 1, 'length_penalty': 'wu_0.5', 'decoding_constraint': 1}, False),
         ('teacher', 'teacher', False)]


def member_weights(family, seed):
    return co.make_weights(family, SMALL['V'], SMALL['E'], SMALL['H'], SMALL['A'], SMALL['F_fc'], SMALL['F_att'], seed=seed, logit_scale=LOGIT_SCALE)


def mix_weights(mix, wname):
    w = WEIGHTS[wname]
    return None if w is None else w[len(MIXES[mix])]


def ref_ensemble(mix, wname):
    from captioning.models.AttEnsemble import AttEnsemble
    models = [ref_model(f, W=member_weights(f, s), **SMALL, **(AOA_EXTRA if f == 'aoa' else {})) for f, s in MIXES[mix]]
    ens = AttEnsemble(models, weights=mix_weights(mix, wname))
    m0 = models[0]
    ens.bos_idx, ens.eos_idx, ens.pad_idx, ens.unk_idx, ens.vocab = m0.bos_idx, m0.eos_idx, m0.pad_idx, m0.unk_idx, m0.vocab
    return ens.eval()


def run_case(ens, fc, att, opts, masked):
    masks = eo.case_masks(B, R) if masked else None
    T = SMALL['T']
    if opts == 'teacher':
        return {'out': ens(fc, att, eo.labels(B, T, SMALL['V'], LABEL_SEED), masks).numpy()}
    seq, lp = ens(fc, att, masks, opt=dict(opts), mode='sample')
    out = {'seq': seq.numpy(), 'logprobs': lp.numpy()}
    if opts.get('beam_size', 1) > 1:
        dseq, dlen, dp = beams_to_arrays(ens.done_beams, opts['beam_size'], T)
        out.update(done_seq=dseq, done_len=dlen, done_p=dp)
    return out


def main():
    out_dir = os.path.join(REPO, 'tests', 'golden')
    _enter_scratch()
    fc, att = co.make_inputs(B, R, SMALL['F_fc'], SMALL['F_att'], seed=INPUT_SEED)
    res = {}
    with torch.no_grad():
        for mix in MIXES:
            for wname in WEIGHTS:
                ens = ref_ensemble(mix, wname)
                for name, opts, masked in CASES:
                    out = run_case(ens, fc, att, opts, masked)
                    for k, v in out.items():
                        res['%s_%s_%s_%s' % (mix, wname, name, k)] = v
                    if 'seq' in out:
                        print(mix, wname, name, 'seq[0]', out['seq'][0].tolist())
    meta = {'cfg': SMALL, 'logit_scale': LOGIT_SCALE, 'aoa_heads': AOA_HEADS, 'B': B, 'R': R, 'input_seed': INPUT_SEED, 'label_seed': LABEL_SEED,
            'mixes': MIXES, 'weights': WEIGHTS, 'cases': CASES}
    np.savez_compressed(os.path.join(out_dir, 'ensemble_small.npz'), meta=np.array(json.dumps(meta)), **res)


if __name__ == '__main__':
    main()
