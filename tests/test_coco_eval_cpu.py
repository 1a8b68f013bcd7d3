"""CPU checks of language evaluation in eval_split: language_eval = 1 still refuses (and names 'device'), a callable still runs, and
'device' on CPU tensors stops at the engine's no-CUDA check instead of falling back; the C entry point is declared."""
import os

import pytest
import torch

from test_eval_cpu import _StubLoader, _StubModel, _crit


class _GtsLoader(_StubLoader):
    """The stub loader with the loader's data['gts']: each image's 0-padded reference rows."""

    def get_batch(self, split):
        data = super().get_batch(split)
        data['gts'] = [self.labels[i['id']][:, 1:-1].numpy() for i in data['infos']]
        return data


def _kwargs(**kw):
    out = {'verbose': False, 'verbose_loss': 1, 'split': 'val', 'dataset': 'coco', 'beam_size': 1, 'sample_n': 1, 'device': 'cpu',
           'num_images': -1}
    out.update(kw)
    return out


def test_language_eval_1_still_refuses_and_names_device(tmp_path, monkeypatch):
    from imagecaptioning.pytorch_b200 import eval_utils as EU
    monkeypatch.chdir(tmp_path)
    with pytest.raises(NotImplementedError, match="'device'"):
        EU.eval_split(_StubModel(6, 12), _crit, _GtsLoader(5, 2, 6, 12), _kwargs(language_eval=1))


def test_language_eval_callable_still_runs(tmp_path, monkeypatch):
    from imagecaptioning.pytorch_b200 import eval_utils as EU
    monkeypatch.chdir(tmp_path)
    seen = {}

    def lang(dataset, preds, preds_n, kw, split):
        seen.update(dataset=dataset, n=len(preds), n_n=len(preds_n), split=split)
        return {'CIDEr': 1.5}

    loss, preds, stats = EU.eval_split(_StubModel(6, 12), _crit, _GtsLoader(5, 2, 6, 12), _kwargs(language_eval=lang))
    assert stats == {'CIDEr': 1.5}
    assert seen == {'dataset': 'coco', 'n': 5, 'n_n': 0, 'split': 'val'}


def test_language_eval_device_on_cpu_tensors_is_refused(tmp_path, monkeypatch):
    from imagecaptioning.pytorch_b200 import eval_utils as EU
    monkeypatch.chdir(tmp_path)
    with pytest.raises(RuntimeError, match='CUDA'):
        EU.eval_split(_StubModel(6, 12), _crit, _GtsLoader(5, 2, 6, 12), _kwargs(language_eval='device'))


def test_coco_scores_refuses_cpu_tensors():
    from imagecaptioning.pytorch_b200 import eval_multi
    with pytest.raises(RuntimeError, match='CUDA'):
        eval_multi.coco_scores(torch.ones(2, 4, dtype=torch.long), [torch.ones(1, 4).numpy()] * 2)
    with pytest.raises(RuntimeError, match='CUDA'):
        eval_multi.eval_oracle(torch.ones(4, 4, dtype=torch.long), [torch.ones(1, 4).numpy()] * 2, 2)


def test_coco_scores_entry_point_is_declared():
    from imagecaptioning.pytorch_b200 import _lib
    assert 'capb200_coco_scores' in _lib.SIGNATURES
    header = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'include', 'capb200.h')
    with open(header) as f:
        assert 'int capb200_coco_scores(' in f.read()
