"""Language evaluation on the device (csrc/coco_eval.cu) against the live coco-caption scorers' values in tests/golden/coco_eval.npz
(written by tests/make_coco_eval_golden.py): every per-caption and overall BLEU-1..4, ROUGE-L and CIDEr within 1e-9 on the small, 256-token,
5000-image and per_image = 5 cases; eval_split(language_eval='device') against the golden scores of its predictions, with predictions and
loss identical to a language_eval = 0 run; the sample_n > 1 and eval_oracle keys; and the refusals."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'coco_eval.npz')
CASES = ('small', 'long', 'split', 'oracle')
METRICS = ('Bleu_1', 'Bleu_2', 'Bleu_3', 'Bleu_4', 'ROUGE_L', 'CIDEr')
TOL = 1e-9


@pytest.fixture(scope='module')
def b200():
    import __graft_entry__ as ge
    ge.build()
    import imagecaptioning.pytorch_b200 as b
    return b


def _case(g, name):
    counts = g[name + '_nrefs']
    refs = g[name + '_refs']
    at = np.concatenate([[0], np.cumsum(counts)])
    gts = [refs[at[i]:at[i + 1]] for i in range(len(counts))]
    return torch.from_numpy(g[name + '_seq'].astype(np.int64)).cuda(), gts, int(g[name + '_per'])


def _close(got, want, tol=TOL):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape
    assert np.abs(got - want).max(initial=0.0) <= tol, np.abs(got - want).max()


@pytest.mark.parametrize('name', CASES)
def test_scores_match_coco_caption(b200, name):
    g = np.load(GOLD)
    seq, gts, per = _case(g, name)
    ids = [1000 + i for i in range(len(gts))]
    out = b200.eval_multi.coco_scores(seq, gts, per_image=per, image_ids=ids)
    rounds = [out['overall']] if per == 1 else out['overall']
    _close([[r[m] for m in METRICS] for r in rounds], g[name + '_overall'])
    caps = [out['imgToEval'][k] for k in ids]
    caps = [c for cs in caps for c in (cs if per > 1 else [cs])]
    assert all(c['image_id'] == ids[i // per] for i, c in enumerate(caps))
    _close([[c['Bleu_%d' % (k + 1)] for k in range(4)] for c in caps], g[name + '_bleu'])
    _close([c['ROUGE_L'] for c in caps], g[name + '_rouge'])
    _close([c['CIDEr'] for c in caps], g[name + '_cider'])


def test_oracle_matches_eval_oracle(b200):
    g = np.load(GOLD)
    seq, gts, per = _case(g, 'oracle')
    out = b200.eval_multi.eval_oracle(seq, gts, per)
    _close([out['overall']['oracle_' + m] for m in METRICS], g['oracle_oracle'])
    _close([out['overall']['avg_' + m] for m in METRICS], g['oracle_avg'])
    assert list(out['ImgToEval']) == list(range(len(gts)))


def test_repeat_calls_are_bitwise_equal(b200):
    g = np.load(GOLD)
    seq, gts, _ = _case(g, 'split')
    a = b200.eval_multi._coco_device(seq, gts, 1)
    b = b200.eval_multi._coco_device(seq, gts, 1)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))


def test_refusals(b200):
    g = np.load(GOLD)
    seq, gts, _ = _case(g, 'small')
    with pytest.raises(ValueError, match='reference'):
        b200.eval_multi.coco_scores(seq, gts[:-1] + [gts[-1][:0]])
    with pytest.raises(ValueError):
        b200.eval_multi.coco_scores(seq, gts[:-1])
    with pytest.raises(RuntimeError, match='CUDA'):
        b200.eval_multi.coco_scores(seq.cpu(), gts)
    long_seq = torch.ones(len(gts), 257, dtype=torch.long, device='cuda')
    with pytest.raises(RuntimeError, match='256'):
        b200.eval_multi.coco_scores(long_seq, gts)
    long_ref = [np.ones((1, 257), np.int32)] * len(gts)
    with pytest.raises(RuntimeError, match='256'):
        b200.eval_multi.coco_scores(seq, long_ref)


# ---- eval_split with language_eval = 'device': a stub model that emits the golden oracle case's captions

class _Loader:
    """The slice of the reference loader eval_split uses, with data['gts']: image i's features hold i."""

    def __init__(self, gts, batch):
        self.gts, self.batch, self.pos, self.n = gts, batch, 0, len(gts)

    def reset_iterator(self, split):
        self.pos = 0

    def get_batch(self, split):
        ix = [(self.pos + i) % self.n for i in range(self.batch)]
        wrapped = self.pos + self.batch >= self.n
        self.pos = (self.pos + self.batch) % self.n
        fc = torch.tensor(ix, dtype=torch.float32)[:, None].repeat(1, 4)
        labels = torch.zeros(len(ix), 1, 18, dtype=torch.long)
        labels[:, 0, 1:17] = torch.from_numpy(np.stack([self.gts[i][0] for i in ix]).astype(np.int64))
        return {'fc_feats': fc, 'att_feats': fc[:, None, :], 'labels': labels, 'masks': torch.ones(len(ix), 1, 18), 'att_masks': None,
                'gts': [self.gts[i] for i in ix], 'infos': [{'id': 500 + i, 'file_path': 'img%d.jpg' % i} for i in ix],
                'bounds': {'it_pos_now': self.pos, 'it_max': self.n, 'wrapped': wrapped}}


class _Model(torch.nn.Module):
    """Greedy captions: caption 0 of each image's golden set; sample_n = n: the image's n golden captions."""

    def __init__(self, caps, per, V1):
        super().__init__()
        self.caps, self.per, self.V1 = caps, per, V1
        self.vocab = {str(i): 'w%d' % i for i in range(1, V1)}
        self.w = torch.nn.Parameter(torch.randn(4, 16 * 8, generator=torch.Generator().manual_seed(3)))
        self.done_beams = []

    def _lp(self, fc, seq):
        small = torch.log_softmax((fc[:, :4] @ self.w.to(fc.device)).view(-1, 16, 8), 2)
        lp = torch.full((fc.shape[0], 16, self.V1), -30.0, device=fc.device)
        lp[:, :, :8] = small
        return lp.scatter(2, seq.unsqueeze(2), small[:, :, :1])

    def forward(self, fc_feats, att_feats, third, *rest, **kw):
        idx = fc_feats[:, 0].long()
        if kw.get('mode', 'forward') == 'sample':
            n = kw.get('opt', {}).get('sample_n', 1)
            rows = (idx[:, None] * self.per + torch.arange(n, device=idx.device)).reshape(-1)
            seq = self.caps.to(idx.device)[rows]
            return seq, self._lp(fc_feats.repeat_interleave(n, 0), seq)
        return self._lp(fc_feats, self.caps.to(idx.device)[idx * self.per])[:, :third.shape[-1]]


def _crit(lp, target, mask):
    target, mask = target.reshape(-1, target.shape[-1])[:, :lp.shape[1]], mask.reshape(-1, mask.shape[-1])[:, :lp.shape[1]]
    return -(lp.gather(2, target.unsqueeze(2)).squeeze(2) * mask).sum() / mask.sum()


def _run(b200, g, tmp_path, monkeypatch, batch, **kw):
    monkeypatch.chdir(tmp_path)
    _, gts, per = _case(g, 'oracle')
    caps = torch.from_numpy(g['oracle_seq'].astype(np.int64))
    kwargs = {'verbose': False, 'verbose_loss': 1, 'split': 'val', 'dataset': 'coco', 'beam_size': 1, 'sample_n': 1, 'num_images': -1,
              'id': 'coco_eval_test'}
    kwargs.update(kw)
    return b200.eval_utils.eval_split(_Model(caps, per, 9488).cuda(), _crit, _Loader(gts, batch), kwargs)


@pytest.mark.parametrize('batch', [20, 25])           # 25 wraps past the split's 60 images: the last batch is trimmed
def test_eval_split_device_language_eval(b200, tmp_path, monkeypatch, batch):
    g = np.load(GOLD)
    loss0, preds0, stats0 = _run(b200, g, tmp_path, monkeypatch, batch, language_eval=0)
    saved0 = torch.load(os.path.join(tmp_path, 'eval_results', '.saved_pred_coco_eval_test_val.pth'))
    loss, preds, stats = _run(b200, g, tmp_path, monkeypatch, batch, language_eval='device')
    saved = torch.load(os.path.join(tmp_path, 'eval_results', '.saved_pred_coco_eval_test_val.pth'))
    assert stats0 is None
    assert loss == loss0 and preds == preds0 and saved == saved0
    assert len(preds) == 60
    assert list(stats) == list(METRICS) + ['perplexity', 'entropy', 'bad_count_rate']
    _close([stats[m] for m in METRICS], g['oracle_overall'][0])
    assert stats['perplexity'] == sum(p['perplexity'] for p in preds) / len(preds)
    assert stats['entropy'] == sum(p['entropy'] for p in preds) / len(preds)
    assert stats['bad_count_rate'] == 0.0                  # 'w<id>' words are never bad endings


def test_eval_split_device_sample_n_and_oracle(b200, tmp_path, monkeypatch):
    g = np.load(GOLD)
    loss0, preds0, _ = _run(b200, g, tmp_path, monkeypatch, 20, language_eval=0, sample_n=5)
    loss, preds, stats = _run(b200, g, tmp_path, monkeypatch, 20, language_eval='device', sample_n=5, eval_oracle=1)
    assert loss == loss0 and preds == preds0
    _close([stats[m] for m in METRICS], g['oracle_overall'][0])
    for m in ('Div1', 'Div2', 'gDiv1', 'mBLeu_1', 'mBLeu_4', 'self_cider'):
        assert np.isfinite(stats[m]), m
    _close([stats['oracle_' + m] for m in METRICS], g['oracle_oracle'])
    _close([stats['avg_' + m] for m in METRICS], g['oracle_avg'])
    _, _, plain = _run(b200, g, tmp_path, monkeypatch, 20, language_eval='device', sample_n=5)
    assert not any(k.startswith(('oracle_', 'avg_')) for k in plain) and 'Div1' in plain
