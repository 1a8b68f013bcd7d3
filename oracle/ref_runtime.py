"""Runs the UNMODIFIED reference (the verbatim copy under oracle/_ref/, see oracle/build_ref.py) on the host cores.

Test infrastructure only: imported by tests/, oracle/make_golden.py and bench.py's CPU arms ("cpu_baseline.kind": "reference"),
never by the product package.  The reference resolves ``cider`` / ``coco-caption`` / ``data/<df>.p`` relative to the working directory
(captioning/utils/rewards.py:12,15; cider/pyciderevalcap/ciderD/ciderD_scorer.py:109), so ``enter()`` switches to a scratch directory
that holds those names as symlinks into oracle/_ref/ plus a writable ``data/``.
"""
from __future__ import annotations

import argparse
import os
import pickle
import sys
import tempfile
from collections import defaultdict

HERE = os.path.dirname(os.path.abspath(__file__))
_REF_COPY = os.path.join(HERE, '_ref')
_state = {'scratch': None, 'root': None}


def available() -> bool:
    return os.path.isdir(os.path.join(_REF_COPY, 'captioning'))


def root() -> str:
    """oracle/_ref, the copy oracle/build_ref.py makes."""
    return _REF_COPY


def enter() -> str:
    """Idempotent: chdir into a scratch directory wired to the reference copy and put the copy on sys.path."""
    if _state['scratch'] is not None:
        os.chdir(_state['scratch'])
        return _state['scratch']
    if not available():
        raise RuntimeError('the reference copy oracle/_ref/ is missing: run python oracle/build_ref.py where the reference is checked out')
    r = root()
    d = tempfile.mkdtemp(prefix='refcwd_')
    os.symlink(os.path.join(r, 'cider'), os.path.join(d, 'cider'))
    os.symlink(os.path.join(r, 'coco-caption'), os.path.join(d, 'coco-caption'))
    os.makedirs(os.path.join(d, 'data'))
    os.chdir(d)
    sys.dont_write_bytecode = True
    if r not in sys.path:
        sys.path.insert(0, r)
    _state['scratch'], _state['root'] = d, r
    return d


def model_opt(family, V, E, H, A, F_fc, F_att, T, **extra):
    opt = argparse.Namespace(vocab_size=V, input_encoding_size=E, rnn_size=H, num_layers=1, drop_prob_lm=0.5, max_length=T, seq_length=T,
                             fc_feat_size=F_fc, att_feat_size=F_att, att_hid_size=A, vocab={str(i): 'w%d' % i for i in range(1, V + 1)},
                             caption_model=family, use_bn=0, logit_layers=1)
    for k, v in extra.items():
        setattr(opt, k, v)
    return opt


FAMILY_EXTRA = {
    'aoa': dict(num_layers=2, refine=1, refine_aoa=1, use_ff=0, decoder_type='AoA', use_multi_head=2, multi_head_scale=1, mean_feats=1, ctx_drop=1,
                dropout_aoa=0.3),
}


def model(family, V, E, H, A, F_fc, F_att, T, W, **extra):
    """The reference's own nn.Module (captioning.models.setup) carrying the state dict ``W``, in eval mode."""
    enter()
    import captioning.models as M
    m = M.setup(model_opt(family, V, E, H, A, F_fc, F_att, T, **extra))
    m.load_state_dict(W, strict=True)
    m.eval()
    return m


def write_df_pickle(name, df, ref_len):
    """data/<name>.p in the format of scripts/prepro_ngrams.py (keys: tuples of strings; the scorer indexes a defaultdict)."""
    d = enter()
    dd = defaultdict(float)
    dd.update({tuple(str(t) for t in k): float(v) for k, v in df.items()})
    with open(os.path.join(d, 'data', name + '.p'), 'wb') as f:
        pickle.dump({'document_frequency': dd, 'ref_len': ref_len}, f, protocol=2)
    return name


def init_scorer(name):
    enter()
    from captioning.utils import rewards as R
    R.CiderD_scorer = None
    R.Cider_scorer = None
    R.Bleu_scorer = None
    R.init_scorer(name)
    return R


def zero_dropout(m):
    """Sets every dropout probability of a reference model to 0 (train mode without RNG), incl. the functional ones."""
    import torch
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
        for attr in ('drop_prob_lm', 'dropout'):
            if isinstance(getattr(mod, attr, None), float):
                setattr(mod, attr, 0.0)
    return m
