"""CPU checks of the caption-set diversity scores: the float64 restatement in diversity_oracle.py reproduces every value the reference
computed for tests/golden/diversity.npz (get_self_cider_scores, my_self_cider, eval_self_cider's steps, compute_div_n /
compute_global_div_n and eval_div_stats' mutual BLEU rounds), the Python entry points refuse bad shapes and corpus tables before any
device work, and the new C ABI symbols are declared with the arity the ctypes layer gives them."""
import os

import numpy as np
import pytest
import torch

import diversity_oracle as O
from helpers import REPO

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'diversity.npz')
NS = (2, 5, 10, 32)


def pickle_df(g, n):
    return {tuple(int(t) for t in row if t != -1): float(v) for row, v in zip(g['dfk_%d' % n], g['dfv_%d' % n])}


@pytest.mark.parametrize('n', NS)
def test_restatement_reproduces_reference(n):
    g = np.load(GOLD)
    s = g['seqs_%d' % n]
    mats, sc = O.self_cider(s, n, pickle_df(g, n), float(g['ref_len_%d' % n]), with_eos=True)
    assert np.abs(mats - g['rmat_%d' % n]).max() < 1e-12
    np.testing.assert_allclose(sc, g['rscore_%d' % n], rtol=0, atol=1e-12)
    df, ref_len = O.document_frequency(g['refs_%d' % n], with_eos=False)
    mats, sc = O.self_cider(s, n, df, ref_len, with_eos=False)
    assert np.abs(mats - g['emat_%d' % n]).max() < 1e-12
    np.testing.assert_allclose(sc, g['escore_%d' % n], rtol=0, atol=1e-12)
    assert np.array_equal(O.div_n(s, n, 1), g['adiv1_%d' % n]) and np.array_equal(O.div_n(s, n, 2), g['adiv2_%d' % n])
    assert O.div_n(s, n, 1).mean() == g['div1_%d' % n] and O.global_div_1(s) == g['gdiv1_%d' % n]
    all_scrs, scrperimg = O.mutual_bleu(s, n)
    assert np.abs(all_scrs - g['mbleu_%d' % n]).max() < 1e-12 and np.abs(scrperimg - g['scrperimg_%d' % n]).max() < 1e-12


def test_golden_covers_the_edge_cases():
    g = np.load(GOLD)
    s = g['seqs_5']
    assert (s[:, 0] == 0).any(), 'an empty caption'
    assert (s[:, -1] != 0).any(), 'a caption without a closing 0'
    assert np.isnan(g['escore_5']).any(), 'an image whose captions are all empty'
    assert int(s.max()) == int(g['meta'][0])
    for n in NS:
        rows = [tuple(r) for r in g['seqs_%d' % n]]
        assert len(set(rows)) < len(rows), 'repeated captions'


def test_document_frequency_helper_is_eval_self_ciders_table():
    from imagecaptioning.pytorch_b200 import eval_multi
    g = np.load(GOLD)
    df, ref_len = eval_multi.document_frequency(g['refs_10'])
    want, want_len = O.document_frequency(g['refs_10'], with_eos=False)
    assert df == want and ref_len == want_len == g['refs_10'].shape[0]


@pytest.fixture
def no_device(monkeypatch):
    import imagecaptioning.pytorch_b200 as b200

    def refuse(*a, **k):
        raise AssertionError('device work before the guard')
    monkeypatch.setattr(b200._lib, 'load', refuse)
    monkeypatch.setattr(b200.rewards, 'CiderD_scorer', object.__new__(b200.rewards.CiderDTable))
    return b200


@pytest.mark.parametrize('n, rows, T, match', [(1, 4, 8, 'at least 2'), (0, 4, 8, 'at least 2'), (33, 66, 8, 'at most 32'), (3, 10, 8, 'sets of 3'),
                                               (2, 4, 65, 'between 1 and 64')])
def test_guards_raise_before_device_work(no_device, n, rows, T, match):
    b200 = no_device
    seqs = torch.ones(rows, T, dtype=torch.long)
    with pytest.raises(ValueError, match=match):
        b200.eval_multi.div_stats(seqs, n)
    with pytest.raises(ValueError, match=match):
        b200.eval_multi.self_cider(seqs, n, b200.rewards.CiderD_scorer)
    with pytest.raises(ValueError, match=match):
        b200.rewards.self_cider(seqs, n)
    if n >= 1 and rows % n == 0:
        with pytest.raises(ValueError, match=match):
            b200.rewards.get_self_cider_scores([None] * (rows // n), seqs, None)


def test_corpus_table_refused(no_device):
    b200 = no_device
    corpus = object.__new__(b200.rewards.CorpusCiderDTable)
    seqs = torch.ones(10, 8, dtype=torch.long)
    with pytest.raises(NotImplementedError, match='corpus'):
        b200.eval_multi.self_cider(seqs, 5, corpus)
    b200.rewards.CiderD_scorer = corpus
    with pytest.raises(NotImplementedError, match='corpus'):
        b200.rewards.get_self_cider_scores([None, None], seqs, None)


def test_uninitialised_scorer_refused(no_device):
    b200 = no_device
    b200.rewards.CiderD_scorer = None
    with pytest.raises(RuntimeError, match='init_scorer'):
        b200.rewards.get_self_cider_scores([None, None], torch.ones(10, 8, dtype=torch.long), None)


def test_diversity_entry_points_declared():
    import imagecaptioning.pytorch_b200 as b200
    hdr = open(os.path.join(REPO, 'include', 'capb200.h')).read()
    for name in ('capb200_self_cider', 'capb200_self_cider_div', 'capb200_div_stats'):
        decl = hdr.split(name + '(')[1].split(')')[0]
        assert len(decl.split(',')) == len(b200._lib.SIGNATURES[name][1]), name
    src = open(os.path.join(REPO, 'imagecaptioning.pytorch_b200', 'csrc', 'diversity.cu')).read()
    assert all(k in src for k in ('self_cider_matrix_kernel', 'self_cider_div_kernel', 'div_stats_kernel', 'mutual_bleu_kernel', 'global_div1_kernel'))
