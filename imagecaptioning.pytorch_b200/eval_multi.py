"""Device-side mirror of the diversity half of captioning/utils/eval_multi.py: the scores the reference's projects/Diversity
``only_eval_test_n_*.sh`` scripts compute for the caption sets ``eval_split_n`` generates.

    div_stats(seqs, n)           eval_div_stats      eval_multi.py:121-175   Div-1, Div-2, gDiv-1, mutual BLEU-1..4
    self_cider(seqs, n, table)   eval_self_cider     eval_multi.py:177-217   self-CIDEr matrices and their eigenvalue diversity

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
