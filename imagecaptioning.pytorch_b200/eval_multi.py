"""Device-side mirror of captioning/utils/eval_multi.py: the scores the reference's projects/Diversity ``only_eval_test_n_*.sh`` scripts
compute for the caption sets ``eval_split_n`` generates, and coco-caption's language metrics that eval_utils.language_eval reports.

    div_stats(seqs, n)           eval_div_stats      eval_multi.py:121-175   Div-1, Div-2, gDiv-1, mutual BLEU-1..4
    self_cider(seqs, n, table)   eval_self_cider     eval_multi.py:177-217   self-CIDEr matrices and their eigenvalue diversity
    coco_scores(seq, gts)        COCOEvalCap         eval_utils.py:84-90     BLEU-1..4, ROUGE-L and CIDEr (no METEOR, SPICE or WMD)
    eval_oracle(seqs, gts, n)    eval_oracle         eval_multi.py:71-119    oracle_ / avg_ BLEU-1..4, ROUGE-L and CIDEr of caption sets

``seqs`` are id rows, n consecutive rows per image (2 <= n <= 32, at most 64 tokens), on a CUDA device -- what ``eval_split_n`` returns.
A caption is its ids before the first 0, the words ``decode_sequence`` would print.  The reference runs coco-caption's PTB tokenizer over
those words first; ids of a vocabulary whose words the tokenizer leaves alone score the same.  Each function runs its kernels
(csrc/diversity.cu) and reads everything back in ONE device-to-host transfer; the final means are numpy's, over the same arrays the
reference averages.

The table of ``eval_self_cider`` holds the document frequencies of the split's references (CiderScorer.compute_doc_freq: an n-gram counts
once per image whose references contain it) and ref_len = the number of images:

    table = rewards.CiderDTable(*eval_multi.document_frequency(refs_per_image))

where ``refs_per_image[i]`` is image i's reference id rows.  Any other CiderDTable (a pickle's, through ``rewards.init_scorer``) works too;
a corpus table has no ref_len and is refused.

``coco_scores`` and ``eval_oracle`` (csrc/coco_eval.cu) return exactly what coco-caption's Bleu(4), Rouge() and Cider() return when each
caption is the string of its ids before the first 0 joined by single spaces, against its image's references -- the loader's ``gts`` rows,
cut the same way.  These are NOT the official COCO numbers: coco-caption's PTB tokenizer never sees the annotation text, and the
references are the dataset's label rows, which prepro truncated at max_length and where rare words are UNK.
"""
from __future__ import annotations

from collections import defaultdict
from typing import Dict, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib
from . import rewards

MAX_V1 = 409600          # the largest V + 1 the engine decodes: the default size of gDiv-1's bitmap


def words(row) -> Tuple[int, ...]:
    """The ids of one caption before its first 0."""
    out = []
    for v in row:
        if int(v) == 0:
            break
        out.append(int(v))
    return tuple(out)


def document_frequency(refs_per_image: Sequence) -> Tuple[Dict[Tuple[int, ...], float], int]:
    """(df, ref_len) of eval_self_cider's Cider(df='corpus') after compute_doc_freq over the split's references (eval_multi.py:186-196):
    df[ngram] = number of images whose references hold the 1..4-gram, ref_len = number of images.  ``refs_per_image[i]`` holds image i's
    reference id rows, each cut before its first 0."""
    df: Dict[Tuple[int, ...], float] = defaultdict(float)
    for rows in refs_per_image:
        seen = set()
        for row in rows:
            w = words(row)
            for k in range(1, 5):
                for i in range(len(w) - k + 1):
                    seen.add(w[i:i + k])
        for g in seen:
            df[g] += 1.0
    return dict(df), len(refs_per_image)


def _device_ids(seqs) -> torch.Tensor:
    if not isinstance(seqs, torch.Tensor) or seqs.dim() != 2:
        raise ValueError('seqs must be a 2-D tensor of caption ids')
    if seqs.device.type != 'cuda':
        raise RuntimeError('capb200: the diversity kernels run on CUDA tensors only')
    return seqs.detach().to(torch.long).contiguous()


COCO_METRICS = ('Bleu_1', 'Bleu_2', 'Bleu_3', 'Bleu_4', 'ROUGE_L', 'CIDEr')
_coco_table: Optional[rewards.CorpusCiderDTable] = None


def _coco_device(seq: torch.Tensor, gts: Sequence, per_image: int):
    """(bleu [S, 4], corpus bleu [per_image, 4], rouge [S], cider [S]) as host float64 arrays from one capb200_coco_scores call and one
    device-to-host transfer."""
    global _coco_table
    if not isinstance(seq, torch.Tensor) or seq.dim() != 2:
        raise ValueError('seq must be a 2-D tensor of caption ids')
    if seq.device.type != 'cuda':
        raise RuntimeError('capb200: the caption metrics run on CUDA tensors only')
    rows, T = (int(x) for x in seq.shape)
    n = int(per_image)
    if n < 1 or rows % n:
        raise ValueError('%d captions do not split into %s per image' % (rows, per_image))
    B = rows // n
    if len(gts) != B:
        raise ValueError('%d reference sets for %d images' % (len(gts), B))
    if B == 0:
        raise ValueError('no images to score')
    if any(int(np.asarray(g).shape[0]) == 0 for g in gts):
        raise ValueError('every image needs at least one reference (coco-caption asserts it)')
    ids = seq.detach().to(torch.long).contiguous()
    if _coco_table is None:
        _coco_table = rewards.CorpusCiderDTable()
    refs, offsets, L = rewards.pack_references(gts, ids.device)
    # one float64 buffer: bleu [S, 4], corpus bleu [n, 4], rouge [S], cider [S], then the int32 BLEU statistics [S, 6]
    o_cb, o_r = 4 * rows, 4 * rows + 4 * n
    o_c, o_st = o_r + rows, o_r + 2 * rows
    buf = torch.empty(o_st + 3 * rows, dtype=torch.float64, device=ids.device)
    p = _lib.ptr(buf)
    _lib.check(_lib.load().capb200_coco_scores(_coco_table._h, _lib.ptr(ids), B, n, T, _lib.ptr(refs), _lib.ptr(offsets), L, p, p + 8 * o_cb,
                                               p + 8 * o_r, p + 8 * o_c, p + 8 * o_st, _lib.current_stream()), 'coco_scores')
    host = buf[:o_st].cpu().numpy()
    return host[:o_cb].reshape(rows, 4), host[o_cb:o_r].reshape(n, 4), host[o_r:o_c], host[o_c:o_st]


def _image_keys(B: int, image_ids: Optional[Sequence]):
    if image_ids is None:
        return list(range(B))
    if len(image_ids) != B:
        raise ValueError('%d image ids for %d images' % (len(image_ids), B))
    return list(image_ids)


def coco_scores(seq: torch.Tensor, gts: Sequence, per_image: int = 1, image_ids: Optional[Sequence] = None):
    """COCOEvalCap's ``eval`` and ``imgToEval`` for BLEU-1..4, ROUGE-L and CIDEr (see the module docstring for what is scored):
        {'overall': {'Bleu_1', .., 'Bleu_4', 'ROUGE_L', 'CIDEr'}, 'imgToEval': {image_id: {'image_id', 'Bleu_1', .., 'CIDEr'}}}
    ``seq`` [n_images * per_image, T] on a CUDA device (RuntimeError otherwise), ``gts[i]`` image i's 0-padded reference rows [n_refs, L]
    (the loader's data['gts']); an image without references raises ValueError.  T and L are at most 256.  With per_image > 1 each of
    the per_image rounds (caption j of every image) is scored as its own COCOEvalCap run, as eval_oracle does: 'overall' is then the list
    of the rounds' dicts and every imgToEval entry the list of its captions' dicts.  Image ids default to 0..B-1."""
    bleu, corpus, rouge, cider = _coco_device(seq, gts, per_image)
    n = int(per_image)
    B = bleu.shape[0] // n
    keys = _image_keys(B, image_ids)
    rounds = []
    for j in range(n):
        overall = {'Bleu_%d' % (k + 1): float(corpus[j, k]) for k in range(4)}
        overall['ROUGE_L'] = float(np.mean(rouge[j::n]))
        overall['CIDEr'] = float(np.mean(cider[j::n]))
        rounds.append(overall)
    per_cap = []
    for i in range(B * n):
        d = {'image_id': keys[i // n]}
        d.update({'Bleu_%d' % (k + 1): float(bleu[i, k]) for k in range(4)})
        d.update({'ROUGE_L': float(rouge[i]), 'CIDEr': float(cider[i])})
        per_cap.append(d)
    if n == 1:
        return {'overall': rounds[0], 'imgToEval': {keys[i]: per_cap[i] for i in range(B)}}
    return {'overall': rounds, 'imgToEval': {keys[i]: per_cap[i * n:(i + 1) * n] for i in range(B)}}


def eval_oracle(seqs: torch.Tensor, gts: Sequence, n: int, image_ids: Optional[Sequence] = None):
    """eval_oracle (eval_multi.py:71-119) for BLEU-1..4, ROUGE-L and CIDEr, as its ``out`` dict:
        {'overall': {'oracle_Bleu_1', 'avg_Bleu_1', .., 'oracle_CIDEr', 'avg_CIDEr'}, 'ImgToEval': {image_id: {same keys}}}
    Round j scores caption j of every image against the image's references (coco_scores with per_image = n); oracle_<m> is an image's best
    caption under metric m, avg_<m> the mean over its captions, and 'overall' the mean of both over the images.  ``seqs`` holds n
    consecutive rows per image, in image order (what eval_split_n returns)."""
    bleu, _, rouge, cider = _coco_device(seqs, gts, n)
    n = int(n)
    B = bleu.shape[0] // n
    keys = _image_keys(B, image_ids)
    per_metric = [bleu[:, k] for k in range(4)] + [rouge, cider]
    img = {}
    for i, key in enumerate(keys):
        d = {}
        for name, vals in zip(COCO_METRICS, per_metric):
            caps = vals[i * n:(i + 1) * n].tolist()
            d['oracle_' + name] = max(caps)
            d['avg_' + name] = sum(caps) / len(caps)
        img[key] = d
    first = next(iter(img.values()))
    overall = {m: np.array([v[m] for v in img.values()]).mean() for m in first}
    return {'overall': overall, 'ImgToEval': img}


def div_stats(seqs: torch.Tensor, n: int, vocab_size: Optional[int] = None, image_ids: Optional[Sequence] = None):
    """eval_div_stats (eval_multi.py:121-175) as its ``out`` dict:
        {'overall': {'Div1', 'Div2', 'gDiv1', 'mBLeu_1', .., 'mBLeu_4'},
         'ImgToEval': {image_id: {'mBleu_2': mean over the image's captions, 'individuals': [{'mBleu_2': caption's BLEU-2}, ...]}}}
    Image ids default to 0..B-1.  Ids must lie in [1, vocab_size] (ValueError otherwise, found on the device); vocab_size defaults to the
    largest vocabulary the engine decodes."""
    rows, T = (int(x) for x in seqs.shape)
    n = int(n)
    B = rewards.check_caption_sets(rows, n, T)
    V1 = MAX_V1 if vocab_size is None else int(vocab_size) + 1
    if image_ids is not None and len(image_ids) != B:
        raise ValueError('%d image ids for %d images' % (len(image_ids), B))
    ids = _device_ids(seqs)
    # one float64 buffer: div1 [B], div2 [B], gdiv1 [1], mbleu [n, 4], bleu2 [B, n], then the int32 BLEU statistics [B, n, 6]
    o_div2, o_g, o_mb, o_b2 = B, 2 * B, 2 * B + 1, 2 * B + 1 + 4 * n
    o_st = o_b2 + B * n
    buf = torch.empty(o_st + B * n * 3, dtype=torch.float64, device=ids.device)
    p = _lib.ptr(buf)
    _lib.check(_lib.load().capb200_div_stats(_lib.ptr(ids), B, n, T, V1, p, p + 8 * o_div2, p + 8 * o_g, p + 8 * o_mb, p + 8 * o_b2, p + 8 * o_st,
                                             _lib.current_stream()), 'div_stats')
    host = buf[:o_st].cpu().numpy()
    if host[o_g] < 0:
        raise ValueError('caption ids outside [1, %d]' % (V1 - 1))
    div1, div2 = host[:B], host[o_div2:o_g]
    all_scrs = host[o_mb:o_b2].reshape(n, 4)
    scrperimg = host[o_b2:o_st].reshape(B, n).T                     # [caption, image], as eval_div_stats fills it
    out = {'overall': {'Div1': div1.mean(), 'Div2': div2.mean(), 'gDiv1': float(host[o_g])}}
    for k, score in zip(range(4), all_scrs.mean(axis=0).tolist()):
        out['overall'].update({'mBLeu_%d' % (k + 1): score})
    keys = list(range(B)) if image_ids is None else list(image_ids)
    per_img, per_cap = scrperimg.mean(axis=0).tolist(), scrperimg.T.tolist()
    out['ImgToEval'] = {imgid: {'mBleu_2': per_img[i], 'individuals': [{'mBleu_2': s} for s in per_cap[i]]} for i, imgid in enumerate(keys)}
    return out


def self_cider(seqs: torch.Tensor, n: int, table: rewards.CiderDTable, image_ids: Optional[Sequence] = None):
    """eval_self_cider (eval_multi.py:177-217) as its dict: {'overall': {'self_cider'}, 'imgToEval': {image_id: {'self_cider',
    'self_cider_mat'}}}, with the document frequencies and ref_len of ``table`` (see the module docstring for the split's own table)."""
    rows, T = (int(x) for x in seqs.shape)
    n = int(n)
    B = rewards.check_caption_sets(rows, n, T)
    if image_ids is not None and len(image_ids) != B:
        raise ValueError('%d image ids for %d images' % (len(image_ids), B))
    if table is None:
        raise ValueError('self_cider needs a document-frequency table')
    rewards._self_cider_table(table)
    mats, scores = rewards.self_cider(_device_ids(seqs), n, table, with_eos=False)
    host = torch.cat([mats.reshape(-1), scores]).cpu().numpy()
    mats, sc = host[:B * n * n].reshape(B, n, n), host[B * n * n:]
    keys = list(range(B)) if image_ids is None else list(image_ids)
    img = {k: {'self_cider': sc[i], 'self_cider_mat': mats[i].tolist()} for i, k in enumerate(keys)}
    return {'overall': {'self_cider': np.mean(np.array(sc))}, 'imgToEval': img}
