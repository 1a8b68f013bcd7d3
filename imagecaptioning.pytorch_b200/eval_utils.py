"""Host-side mirror of the evaluation loop around the decode hot path: captioning/utils/eval_utils.py:129-213 (``eval_split``) and the
feature hand-off of captioning/data/dataloader.py:317-332 (``get_batch``).

SURVEY.md section 8(f) rank 4: once the decode itself is fast, the reference's evaluation loop is dominated by host work --
``tensor.to(device)`` from pageable memory on the critical path, one ``.item()`` (a device synchronisation) per caption for the
perplexity and the entropy, one per token in ``decode_sequence``.  This module keeps the reference's contract

    eval_split(model, crit, loader, eval_kwargs) -> (mean loss, predictions, lang_stats)

and its ``predictions`` entries (``image_id``, ``caption``, ``perplexity``, ``entropy``) but

  * ``PrefetchLoader`` pins every batch's tensors and copies batch i+1 host -> device on a side stream while batch i decodes,
  * perplexity / entropy are reduced on the device for the whole batch and fetched with ONE device -> host copy,
  * captions are detokenised by ``utils.decode_sequence`` (one copy per batch).

Language evaluation:
  * ``eval_kwargs['language_eval'] = 'device'`` scores the split on the GPU after the loop (eval_multi.coco_scores, csrc/coco_eval.cu):
    BLEU-1..4, ROUGE-L and CIDEr of every kept caption against its image's ``data['gts']`` rows, plus perplexity, entropy and
    bad_count_rate, under the key names of the reference's language_eval (eval_utils.py:89-121).  With sample_n > 1 the caption sets add
    eval_multi.div_stats' and eval_multi.self_cider's statistics and, with ``eval_kwargs['eval_oracle']``, eval_multi.eval_oracle's.  The
    scores are coco-caption's Bleu(4) / Rouge() / Cider() over the ids joined by spaces, not the official COCO numbers: there is no PTB
    tokenization of the annotation text and the references are the label rows (truncated at max_length, rare words UNK).  METEOR, SPICE,
    WMD, AllSPICE, novel_sentences and vocab_size are absent.
  * ``language_eval = 1`` means the reference's Java tool chain (METEOR / SPICE), which is not run here and raises; pass a callable
    ``(dataset, predictions, n_predictions, eval_kwargs, split) -> stats`` to plug the reference's ``eval_utils.language_eval`` in.
"""
from __future__ import annotations

import os
from typing import Any, Dict, Iterator, Optional, Tuple

import torch

from .utils import decode_sequence

_TENSOR_KEYS = ('fc_feats', 'att_feats', 'labels', 'masks', 'att_masks')


class PrefetchLoader:
    """Iterates ``loader.get_batch(split)`` (the reference's loader API, dataloader.py:317-332) one batch ahead: the tensors of batch i+1
    are pinned and copied to ``device`` on a side stream while the caller still works on batch i.  Yields the loader's dict with the five
    tensor entries replaced by device tensors (``None`` stays ``None``).  On a CPU ``device`` it degrades to a plain pass-through."""

    def __init__(self, loader, split: str, device='cuda', max_batches: Optional[int] = None):
        self.loader, self.split, self.max_batches = loader, split, max_batches
        self.device = torch.device(device)
        self.cuda = self.device.type == 'cuda'
        self.stream = torch.cuda.Stream(device=self.device) if self.cuda else None

    def _stage(self, data: Dict[str, Any]) -> Tuple[Dict[str, Any], Optional[torch.cuda.Event]]:
        if not self.cuda:
            return data, None
        out = dict(data)
        with torch.cuda.stream(self.stream):
            for k in _TENSOR_KEYS:
                t = data.get(k)
                if t is None:
                    continue
                t = torch.as_tensor(t)
                if not t.is_cuda:
                    t = t.pin_memory() if not t.is_pinned() else t
                out[k] = t.to(self.device, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.stream)
        return out, ev

    def __iter__(self) -> Iterator[Dict[str, Any]]:
        n = 0
        nxt = self._stage(self.loader.get_batch(self.split))
        while nxt is not None:
            data, ev = nxt
            n += 1
            wrapped = bool(data.get('bounds', {}).get('wrapped', False))
            more = not wrapped and (self.max_batches is None or n < self.max_batches)
            nxt = self._stage(self.loader.get_batch(self.split)) if more else None      # the copy of batch i+1 overlaps the work on batch i
            if ev is not None:
                cur = torch.cuda.current_stream(self.device)
                cur.wait_event(ev)
                for k in _TENSOR_KEYS:
                    if isinstance(data.get(k), torch.Tensor):
                        data[k].record_stream(cur)
            yield data


def caption_stats(seq: torch.Tensor, seq_logprobs: torch.Tensor):
    """(perplexity [N], entropy [N]) exactly as eval_utils.py:173-174, as device tensors (no host synchronisation)."""
    denom = (seq > 0).to(seq_logprobs).sum(1) + 1
    entropy = -(torch.softmax(seq_logprobs, dim=2) * seq_logprobs).sum(2).sum(1) / denom
    perplexity = -seq_logprobs.gather(2, seq.unsqueeze(2)).squeeze(2).sum(1) / denom
    return perplexity, entropy


def eval_split_n(model, n_predictions, input_data, eval_kwargs: Dict[str, Any] = {}):
    """Contract of captioning/utils/eval_utils.py:230-283: ``sample_n`` captions per image, appended to ``n_predictions``.
    ``sample_n_method`` 'bs' (the sample_n best beams), 'sample' / 'gumbel' / 'top<k>' / 'top<p>' (sample_n draws, with their perplexity:
    read back with ONE transfer for the batch instead of one .item() per caption).  'dbs' is diverse beam search: sample_n groups of
    beam_size beams, one caption per group (each group's best), on the engine for UpDown and AoANet.  The remaining branch is diverse
    sampling (group_size > 1 with beam_size 1), which the engine refuses; the model's own NotImplementedError surfaces.

    Returns the captions' ids, int64 [n_images * sample_n, T] on the model's device, in the order they were appended to ``n_predictions``
    (sample_n consecutive rows per image): ``eval_multi.div_stats`` / ``eval_multi.self_cider`` score them without re-tokenising."""
    verbose = eval_kwargs.get('verbose', True)
    beam_size = eval_kwargs.get('beam_size', 1)
    sample_n = eval_kwargs.get('sample_n', 1)
    sample_n_method = eval_kwargs.get('sample_n_method', 'sample')
    fc_feats, att_feats, att_masks, data = input_data
    kw = dict(eval_kwargs)
    n_images = fc_feats.shape[0]
    if sample_n_method == 'bs':
        kw.update({'sample_n': 1, 'beam_size': sample_n, 'group_size': 1})
        with torch.no_grad():
            model(fc_feats, att_feats, att_masks, opt=kw, mode='sample')
        rows = []
        for k in range(n_images):
            rows.append(torch.stack([model.done_beams[k][_]['seq'] for _ in range(sample_n)]))
            sents = decode_sequence(model.vocab, rows[-1])
            for sent in sents:
                n_predictions.append({'image_id': data['infos'][k]['id'], 'caption': sent})
    elif sample_n_method in ('sample', 'gumbel') or sample_n_method.startswith('top'):
        kw.update({'sample_n': sample_n, 'sample_method': sample_n_method, 'beam_size': 1})
        with torch.no_grad():
            seq, logprobs = model(fc_feats, att_feats, att_masks, opt=kw, mode='sample')
        perplexity = (-logprobs.gather(2, seq.unsqueeze(2)).squeeze(2).sum(1) / ((seq > 0).to(logprobs).sum(1) + 1)).cpu().tolist()
        for k, sent in enumerate(decode_sequence(model.vocab, seq)):
            n_predictions.append({'image_id': data['infos'][k // sample_n]['id'], 'caption': sent, 'perplexity': perplexity[k]})
    elif sample_n_method == 'dbs':
        kw.update({'beam_size': sample_n * beam_size, 'group_size': sample_n})
        with torch.no_grad():
            model(fc_feats, att_feats, att_masks, opt=kw, mode='sample')
        rows = []
        for k in range(n_images):
            rows.append(torch.stack([model.done_beams[k][_]['seq'] for _ in range(0, sample_n * beam_size, beam_size)]))
            sents = decode_sequence(model.vocab, rows[-1])
            for sent in sents:
                n_predictions.append({'image_id': data['infos'][k]['id'], 'caption': sent})
    else:
        kw.update({'sample_method': sample_n_method[1:], 'group_size': sample_n, 'beam_size': 1})
        with torch.no_grad():
            seq, _ = model(fc_feats, att_feats, att_masks, opt=kw, mode='sample')
        for k, sent in enumerate(decode_sequence(model.vocab, seq)):
            n_predictions.append({'image_id': data['infos'][k // sample_n]['id'], 'caption': sent})
    if verbose:
        for entry in sorted(n_predictions[-n_images * sample_n:], key=lambda x: x['image_id']):
            print('image %s: %s' % (entry['image_id'], entry['caption']))
    if sample_n_method in ('bs', 'dbs'):
        T = max(r.shape[1] for r in rows)
        seq = torch.cat([torch.nn.functional.pad(r, (0, T - r.shape[1])) for r in rows])
    return seq


def _pad_cat(chunks):
    T = max(int(c.shape[1]) for c in chunks)
    return torch.cat([torch.nn.functional.pad(c, (0, T - int(c.shape[1]))) for c in chunks])


def count_bad(sen: str) -> int:
    """eval_utils.py:31-36: 1 when the caption's last word is a bad ending."""
    from .models import BAD_ENDINGS
    return 1 if sen.split(' ')[-1] in BAD_ENDINGS else 0


def device_language_eval(predictions, seqs, gts, n_seqs, n_gts, sample_n: int, eval_kwargs: Dict[str, Any]):
    """lang_stats of ``language_eval = 'device'``: the key names of eval_utils.py:89-121 (language_eval) for the metrics computed on the
    device.  ``seqs`` / ``gts``: the id chunks and reference sets of ``predictions``, in their order; ``n_seqs`` / ``n_gts``: the caption
    sets eval_split_n returned and their images' references, in image order."""
    from . import eval_multi, rewards
    out = dict(eval_multi.coco_scores(_pad_cat(seqs), gts, image_ids=[p['image_id'] for p in predictions])['overall'])
    out['perplexity'] = sum([p['perplexity'] for p in predictions]) / len(predictions)
    out['entropy'] = sum([p['entropy'] for p in predictions]) / len(predictions)
    if n_seqs:
        seq_n = _pad_cat(n_seqs)
        out.update(eval_multi.div_stats(seq_n, sample_n)['overall'])
        if eval_kwargs.get('eval_oracle', 0):
            out.update(eval_multi.eval_oracle(seq_n, n_gts, sample_n)['overall'])
        table = rewards.CiderDTable(*eval_multi.document_frequency(n_gts))
        out.update(eval_multi.self_cider(seq_n, sample_n, table)['overall'])
    out['bad_count_rate'] = sum([count_bad(p['caption']) for p in predictions]) / float(len(predictions))
    return out


def eval_split(model, crit, loader, eval_kwargs: Dict[str, Any] = {}):
    """Contract of captioning/utils/eval_utils.py:129-213.  ``crit`` is the XE criterion (LanguageModelCriterion / LabelSmoothing)."""
    verbose = eval_kwargs.get('verbose', True)
    verbose_beam = eval_kwargs.get('verbose_beam', 0)
    verbose_loss = eval_kwargs.get('verbose_loss', 1)
    num_images = eval_kwargs.get('num_images', eval_kwargs.get('val_images_use', -1))
    split = eval_kwargs.get('split', 'val')
    lang_eval = eval_kwargs.get('language_eval', 0)
    dataset = eval_kwargs.get('dataset', 'coco')
    beam_size = eval_kwargs.get('beam_size', 1)
    sample_n = eval_kwargs.get('sample_n', 1)
    remove_bad_endings = eval_kwargs.get('remove_bad_endings', 0)
    os.environ['REMOVE_BAD_ENDINGS'] = str(remove_bad_endings)      # same global configuration channel as the reference (eval_utils.py:139)
    device = eval_kwargs.get('device', 'cuda')
    model.eval()
    loader.reset_iterator(split)
    n, loss, loss_sum, loss_evals = 0, 0.0, 0.0, 1e-8
    predictions, n_predictions = [], []
    on_device = isinstance(lang_eval, str) and lang_eval == 'device'
    lang_seqs, lang_gts, lang_n_seqs, lang_n_gts = [], [], [], []      # what language_eval = 'device' scores after the loop
    for data in PrefetchLoader(loader, split, device):
        n += len(data['infos'])
        fc_feats, att_feats, labels, masks, att_masks = (data[k] for k in _TENSOR_KEYS)
        loss_t = None
        if labels is not None and verbose_loss:
            with torch.no_grad():
                loss_t = crit(model(fc_feats, att_feats, labels[..., :-1], att_masks), labels[..., 1:], masks[..., 1:])
        with torch.no_grad():
            kw = dict(eval_kwargs)
            kw.update({'sample_n': 1})
            seq, seq_logprobs = model(fc_feats, att_feats, att_masks, opt=kw, mode='sample')
            seq = seq.data
            perplexity, entropy = caption_stats(seq, seq_logprobs)
        # one device -> host transfer for the batch's scalars (the reference: 2 .item() per caption + 1 for the loss)
        scal = torch.stack([perplexity, entropy]).double()
        if loss_t is not None:
            scal = torch.cat([scal.reshape(-1), loss_t.reshape(1).double()])
        scal = scal.reshape(-1).cpu().tolist()
        N = seq.shape[0]
        perp, ent = scal[:N], scal[N:2 * N]
        if loss_t is not None:
            loss = scal[2 * N]
            loss_sum += loss
            loss_evals += 1
        if beam_size > 1 and verbose_beam:
            for i in range(fc_feats.shape[0]):
                print('\n'.join([decode_sequence(model.vocab, _['seq'].unsqueeze(0))[0] for _ in model.done_beams[i]]))
                print('--' * 10)
        sents = decode_sequence(model.vocab, seq)
        for k, sent in enumerate(sents):
            entry = {'image_id': data['infos'][k]['id'], 'caption': sent, 'perplexity': perp[k], 'entropy': ent[k]}
            if eval_kwargs.get('dump_path', 0) == 1:
                entry['file_name'] = data['infos'][k]['file_path']
            predictions.append(entry)
            if verbose:
                print('image %s: %s' % (entry['image_id'], entry['caption']))
        if sample_n > 1:
            seq_n = eval_split_n(model, n_predictions, [fc_feats, att_feats, att_masks, data], eval_kwargs)
            if on_device:
                lang_n_seqs.append(seq_n)
                lang_n_gts.extend(data['gts'])
        ix1 = data['bounds']['it_max']
        if num_images != -1:
            ix1 = min(ix1, num_images)
        else:
            num_images = ix1
        for _ in range(n - ix1):
            predictions.pop()
        if on_device:                   # the captions and references of the predictions kept, trimmed as predictions was
            lang_seqs.append(seq)
            lang_gts.extend(data['gts'])
            del lang_gts[len(predictions):]
            extra = sum(int(c.shape[0]) for c in lang_seqs) - len(predictions)
            while extra > 0:
                last = lang_seqs.pop()
                if int(last.shape[0]) > extra:
                    lang_seqs.append(last[:int(last.shape[0]) - extra])
                extra -= min(extra, int(last.shape[0]))
        if verbose:
            print('evaluating validation preformance... %d/%d (%f)' % (n, ix1, loss))
        if num_images >= 0 and n >= num_images:
            break

    lang_stats = None
    if len(n_predictions) > 0 and 'perplexity' in n_predictions[0]:
        n_predictions = sorted(n_predictions, key=lambda x: x['perplexity'])
    if 'id' in eval_kwargs:         # the reference's side effect (eval_utils.py:217-219): language_eval and tools/eval.py read this file back
        os.makedirs('eval_results', exist_ok=True)
        torch.save((predictions, n_predictions), os.path.join('eval_results/', '.saved_pred_' + eval_kwargs['id'] + '_' + split + '.pth'))
    if callable(lang_eval):
        lang_stats = lang_eval(dataset, predictions, n_predictions, eval_kwargs, split)
    elif on_device:
        lang_stats = device_language_eval(predictions, lang_seqs, lang_gts, lang_n_seqs, lang_n_gts, sample_n, eval_kwargs)
    elif lang_eval == 1:
        raise NotImplementedError("language_eval = 1 runs the reference's Java tool chain (METEOR, SPICE): pass eval_kwargs['language_eval'] = "
                                  "'device' for BLEU, ROUGE-L and CIDEr on the GPU, or eval_utils.language_eval")
    model.train()
    return loss_sum / loss_evals, predictions, lang_stats
