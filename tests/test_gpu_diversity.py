"""The diversity kernels (csrc/diversity.cu) against the reference's own values in tests/golden/diversity.npz: self-CIDEr matrices and
eigenvalue scores in both caption forms within 1e-6, Div-1 / Div-2 / gDiv-1 exactly, mutual BLEU within 1e-6; the eigenvalue kernel
against numpy's eigvalsh on asymmetric matrices (lower triangle); a 5000 x 10 set in one call, bitwise the same on a second call; and
eval_split_n's returned ids against its captions."""
import argparse

import numpy as np
import pytest
import torch

import diversity_oracle as O

pytestmark = pytest.mark.gpu

from test_diversity_cpu import GOLD, NS, pickle_df     # noqa: E402


@pytest.fixture(scope='module')
def b200():
    import __graft_entry__ as ge
    ge.build()
    import imagecaptioning.pytorch_b200 as b
    return b


def _close(got, want, tol=1e-6):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape
    assert np.array_equal(np.isnan(got), np.isnan(want))
    ok = ~np.isnan(want)
    assert np.abs(got[ok] - want[ok]).max(initial=0.0) <= tol, np.abs(got[ok] - want[ok]).max()


@pytest.mark.parametrize('n', NS)
def test_self_cider_reward_form_matches_reference(b200, n):
    g = np.load(GOLD)
    seqs = torch.from_numpy(g['seqs_%d' % n]).cuda()
    table = b200.rewards.CiderDTable(pickle_df(g, n), float(g['ref_len_%d' % n]))
    b200.rewards.reset_scorer()
    b200.rewards.init_scorer(table)
    try:
        B = seqs.shape[0] // n
        scores = b200.rewards.get_self_cider_scores([None] * B, seqs, argparse.Namespace())
        assert scores.dtype == torch.float64 and scores.is_cuda and scores.shape == (B,)
        _close(scores.cpu().numpy(), g['rscore_%d' % n])
        mats, _ = b200.rewards.self_cider(seqs, n)
        _close(mats.cpu().numpy(), g['rmat_%d' % n])
    finally:
        b200.rewards.reset_scorer()


@pytest.mark.parametrize('n', NS)
def test_eval_self_cider_matches_reference(b200, n):
    g = np.load(GOLD)
    table = b200.rewards.CiderDTable(*b200.eval_multi.document_frequency(g['refs_%d' % n]))
    out = b200.eval_multi.self_cider(torch.from_numpy(g['seqs_%d' % n]).cuda(), n, table, image_ids=[100 + i for i in range(len(g['escore_%d' % n]))])
    imgs = out['imgToEval']
    assert list(imgs) == [100 + i for i in range(len(imgs))]
    _close([imgs[k]['self_cider'] for k in imgs], g['escore_%d' % n])
    _close(np.array([imgs[k]['self_cider_mat'] for k in imgs]), g['emat_%d' % n])
    _close(out['overall']['self_cider'], g['eself_%d' % n])


@pytest.mark.parametrize('n', NS)
def test_div_stats_match_reference(b200, n):
    g = np.load(GOLD)
    out = b200.eval_multi.div_stats(torch.from_numpy(g['seqs_%d' % n]).cuda(), n, vocab_size=int(g['meta'][0]))
    ov = out['overall']
    assert ov['Div1'] == g['div1_%d' % n] and ov['Div2'] == g['div2_%d' % n] and ov['gDiv1'] == g['gdiv1_%d' % n]
    mb = g['mbleu_%d' % n].mean(axis=0)
    _close([ov['mBLeu_%d' % (k + 1)] for k in range(4)], mb)
    spi = g['scrperimg_%d' % n]
    imgs = out['ImgToEval']
    _close([imgs[i]['mBleu_2'] for i in range(spi.shape[1])], spi.mean(axis=0))
    _close([[d['mBleu_2'] for d in imgs[i]['individuals']] for i in range(spi.shape[1])], spi.T)


def test_ids_outside_the_vocabulary_raise(b200):
    g = np.load(GOLD)
    with pytest.raises(ValueError, match='outside'):
        b200.eval_multi.div_stats(torch.from_numpy(g['seqs_5']).cuda(), 5, vocab_size=100)


@pytest.mark.parametrize('n', [2, 3, 7, 16, 32])
def test_eigenvalue_diversity_reads_the_lower_triangle(b200, n):
    rng = np.random.RandomState(n)
    B = 40
    x = rng.rand(B, n, 6)
    mats = 10.0 * np.einsum('bik,bjk->bij', x, x) / 6.0
    mats[1:8] += np.triu(rng.rand(n, n), 1) * 3.0                     # upper triangles eigvalsh never reads
    mats[8] = 10.0                                                      # rank one
    mats[9] = np.diag(rng.rand(n)) * 10.0                               # already diagonal
    mats[10] = 0.0                                                      # nothing: nan, as numpy gives
    mats[11] = -np.eye(n)                                               # negative eigenvalues clip to 0
    mats[11, 0, 0] = 4.0
    want = []
    for m in mats:
        with np.errstate(divide='ignore', invalid='ignore'):
            want.append(O.get_div(m))
    d = torch.from_numpy(mats).cuda()
    out = torch.empty(B, dtype=torch.float64, device='cuda')
    lib = b200._lib.load()
    b200._lib.check(lib.capb200_self_cider_div(b200._lib.ptr(d), B, n, b200._lib.ptr(out), b200._lib.current_stream()), 'self_cider_div')
    _close(out.cpu().numpy(), np.array(want))


def test_5000_images_of_10_in_one_call(b200):
    n, B, T, V = 10, 5000, 16, 9487
    rng = np.random.RandomState(5)
    seqs = np.zeros((B * n, T), np.int64)
    lens = rng.randint(0, T + 1, size=B * n)
    for r in range(B * n):
        pool = rng.randint(1, V + 1, size=12)
        seqs[r, :lens[r]] = pool[rng.randint(0, 12, size=lens[r])] if r % 2 else rng.randint(1, 60, size=lens[r])
    refs = [seqs[i * n:i * n + 3] for i in range(B)]
    df, ref_len = O.document_frequency(refs, with_eos=True)
    table = b200.rewards.CiderDTable(df, ref_len)
    d = torch.from_numpy(seqs).cuda()
    m1, s1 = (t.clone() for t in b200.rewards.self_cider(d, n, table))
    m2, s2 = b200.rewards.self_cider(d, n, table)
    torch.cuda.synchronize()
    assert torch.equal(m1, m2) and torch.equal(s1, s2)
    o1 = b200.eval_multi.div_stats(d, n, vocab_size=V)
    o2 = b200.eval_multi.div_stats(d, n, vocab_size=V)
    assert o1['overall'] == o2['overall']
    assert all(o1['ImgToEval'][i]['mBleu_2'] == o2['ImgToEval'][i]['mBleu_2'] for i in range(B))
    pick = [0, 1, 2, 1234, 4999]
    sub = np.concatenate([seqs[i * n:(i + 1) * n] for i in pick])
    wm, ws = O.self_cider(sub, n, df, ref_len, with_eos=True)
    _close(m1.cpu().numpy()[pick], wm)
    _close(s1.cpu().numpy()[pick], ws)
    assert o1['overall']['Div1'] == O.div_n(seqs, n, 1).mean() and o1['overall']['gDiv1'] == O.global_div_1(seqs)
    all_scrs, scrperimg = O.mutual_bleu(seqs, n)
    _close([o1['overall']['mBLeu_%d' % (k + 1)] for k in range(4)], all_scrs.mean(axis=0))
    _close([o1['ImgToEval'][i]['mBleu_2'] for i in pick], scrperimg[:, pick].mean(axis=0))


@pytest.mark.parametrize('method', ['sample', 'bs'])
def test_eval_split_n_returns_the_ids_of_its_captions(b200, method):
    from helpers import build_pair
    from oracle import caption_oracle as co
    cfg = dict(V=60, E=32, H=32, A=16, F_fc=48, F_att=48, T=8)
    fc, att = co.make_inputs(4, 7, 48, 48, seed=11)
    model, _ = build_pair('updown', seed=11, logit_scale=20.0, mode='simt_fp32', **cfg)
    preds = []
    data = {'infos': [{'id': 100 + i} for i in range(4)]}
    seq = b200.eval_utils.eval_split_n(model, preds, (fc.cuda(), att.cuda(), None, data),
                                       {'sample_n_method': method, 'sample_n': 3, 'beam_size': 3, 'verbose': False})
    assert seq.shape[0] == 12 and seq.dtype == torch.long and seq.is_cuda
    assert b200.decode_sequence(model.vocab, seq) == [p['caption'] for p in preds]
    out = b200.eval_multi.div_stats(seq, 3, vocab_size=cfg['V'])
    assert out['overall']['Div1'] == O.div_n(seq.cpu().numpy(), 3, 1).mean()
