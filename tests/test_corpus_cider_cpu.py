"""CPU checks of corpus-mode CIDEr-D (init_scorer('corpus') -> CiderD(df='corpus')): a numpy restatement of its document frequencies and
ref_len reproduces the reference's own rewards and scores stored in tests/golden/corpus_cider.npz -- df counts the scored hypotheses (crefs
entries) whose image has the n-gram among its references, each image n + 1 times for get_self_critical_reward and n times for get_scores,
ref_len = log(number of entries) -- and init_scorer('corpus') reads no file."""
import builtins
import os

import numpy as np
import pytest

from oracle import ciderd_oracle as cdo

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'corpus_cider.npz')


def corpus_df(gts, entries_per_image):
    """Corpus-mode document frequencies and the entry count ref_len is the log of."""
    df, images = cdo.build_document_frequency(gts)
    return {k: v * entries_per_image for k, v in df.items()}, images * entries_per_image


def test_corpus_restatement_matches_reference():
    g = np.load(GOLD)
    V, B, n, T = (int(x) for x in g['meta'])
    gts = [g['gts'][i] for i in range(B)]
    assert np.asarray(g['weights'])[0].tolist() == [1.0, 0.0]
    df, entries = corpus_df(gts, n + 1)
    assert entries == B * (n + 1)
    reward, _ = cdo.self_critical_reward(g['greedy'], gts, g['sampled'], df, entries)
    assert np.abs(reward - g['reward_0']).max() < 1e-12
    df, entries = corpus_df(gts, n)
    scores = cdo.get_scores(gts, g['sampled'], df, entries)
    assert np.abs(scores - g['scores_0']).max() < 1e-12
    # the entry count matters: the image-count table of a pickle gives other values
    df1, images = cdo.build_document_frequency(gts)
    assert np.abs(cdo.get_scores(gts, g['sampled'], df1, images) - g['scores_0']).max() > 1e-3
    assert np.abs(g['reward_0']).max() > 1e-2


def test_init_scorer_corpus_reads_no_file(monkeypatch):
    import imagecaptioning.pytorch_b200 as b200
    b200.rewards.reset_scorer()

    def no_files(*a, **k):
        raise AssertionError('init_scorer(corpus) opened a file')
    monkeypatch.setattr(builtins, 'open', no_files)
    try:
        b200.rewards.init_scorer('corpus')
    except RuntimeError as e:          # without a GPU the device table cannot be created: the CUDA error, not a missing data/corpus.p
        assert 'corpus.p' not in str(e)
    else:
        assert isinstance(b200.rewards.CiderD_scorer, b200.rewards.CorpusCiderDTable)
    finally:
        b200.rewards.reset_scorer()


def test_corpus_entry_points_in_header():
    import imagecaptioning.pytorch_b200 as b200
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'include', 'capb200.h')).read()
    for name in ('capb200_cider_corpus_table_create', 'capb200_cider_table_reserve', 'capb200_cider_table_is_corpus'):
        decl = hdr.split(name + '(')[1].split(')')[0]
        nargs = 0 if decl.strip() == 'void' else len(decl.split(','))
        assert nargs == len(b200._lib.SIGNATURES[name][1]), name
