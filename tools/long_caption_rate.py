"""Cost of long captions: the Transformer decode past 31 positions, the SCST steps past 64 tokens, and the long reward kernels.

1. Transformer (6 + 6 layers, d_model 512, 8 heads, V = 9487) beam-5 decode of 10 images at 36 regions for seq_length T in
   {20, 31, 32, 64, 128, 256}: up to 31 the decoder self-attention runs its one-lane-per-position kernel, from 32 on the chunked one.
2. The Transformer and the UpDown (E = H = 1000, A = 512) self-critical steps, 10 images x 5 samples, at T in {20, 64, 128}; the second
   call of a shape captures the step graph and later calls replay it.
3. The standalone weighted reward (0.7 CIDEr-D + 0.3 BLEU-4, greedy baseline: 50 samples + 10 greedy captions, 5 references per image) at
   caption / reference widths 64 (the original kernels), 65 and 256 (the long ones).  CUDA events around `--launches` calls.
The word-0 (EOS) bias of every model is lowered by 30, so every caption runs the full T.  Steps and decodes are timed with a host clock
around `--steps` calls ending in a device synchronise.  Prints one JSON line with the card name and power limit read in the same run.

    python tools/long_caption_rate.py [--steps 3] [--repeats 3] [--launches 50]
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tools'))

from dbs_rate import device_info            # noqa: E402
from large_vocab_rate import timed          # noqa: E402

B, N_PER, R, V = 10, 5, 36, 9487
TFM = dict(V=V, E=512, H=2048, A=6, F_fc=2048, F_att=2048)
UPDOWN = dict(V=V, E=1000, H=1000, A=512, F_fc=2048, F_att=2048)


def long_refs(n_images, width, seed):
    rng = np.random.RandomState(seed)
    out = []
    for _ in range(n_images):
        rows = np.zeros((5, width), np.int64)
        for j in range(5):
            ln = rng.randint(width // 2, width + 1)
            rows[j, :ln] = np.minimum(rng.zipf(1.3, size=ln), V)
        out.append(rows)
    return out


def model(family, T, cfg):
    from imagecaptioning.pytorch_b200 import synthetic as syn
    m = syn.build_model(family, seed=1234, logit_scale=3.0, mode='tc_f16x3', device=torch.device('cuda:0'), heads=8, T=T, **cfg)
    key = 'model.generator.proj.bias' if family == 'transformer' else 'logit.bias'
    with torch.no_grad():
        m.state_dict()[key][0] -= 30.0          # before the first call, which binds the weights
    return m


def decode_table(steps, repeats):
    from imagecaptioning.pytorch_b200 import synthetic as syn
    fc, att = (t.cuda() for t in syn.make_inputs(B, R, TFM['F_fc'], TFM['F_att'], seed=1))
    out = {}
    for T in (20, 31, 32, 64, 128, 256):
        m = model('transformer', T, TFM)

        def run():
            with torch.no_grad():
                seq, _ = m(fc, att, None, opt={'beam_size': 5, 'sample_n': 1}, mode='sample')
            return seq
        out['transformer beam5 decode B=10 T=%d' % T] = timed(run, steps, 1, repeats)
        del m
        torch.cuda.empty_cache()
    return out


def scst_table(steps, repeats):
    import imagecaptioning.pytorch_b200 as b200
    from imagecaptioning.pytorch_b200 import synthetic as syn
    table = b200.rewards.CiderDTable(*syn.document_frequency(syn.make_refs(200, V, seed=4) + long_refs(100, 128, seed=5)))
    fc, att = (t.cuda() for t in syn.make_inputs(B, R, 2048, 2048, seed=2))
    out = {}
    for family, cfg in (('transformer', TFM), ('updown', UPDOWN)):
        for T in (20, 64, 128):
            m = model(family, T, cfg)
            m.train()
            refs = long_refs(B, T, seed=T)
            out['%s scst_step 10x5 T=%d' % (family, T)] = timed(lambda: m.scst_step(fc, att, refs, table, N_PER), steps, 2, repeats)
            del m
            torch.cuda.empty_cache()
    return out


def reward_table(launches, repeats):
    import imagecaptioning.pytorch_b200 as b200
    from imagecaptioning.pytorch_b200 import synthetic as syn
    b200.rewards.reset_scorer()
    b200.rewards.init_scorer(b200.rewards.CiderDTable(*syn.document_frequency(syn.make_refs(200, V, seed=4) + long_refs(100, 256, seed=6))))
    rng = np.random.RandomState(3)
    out = {}
    for width in (64, 65, 256):
        refs = long_refs(B, width, seed=width)
        sampled = torch.from_numpy(np.minimum(rng.zipf(1.3, size=(B * N_PER, width)), V)).cuda()
        greedy = torch.from_numpy(np.minimum(rng.zipf(1.3, size=(B, width)), V)).cuda()

        def call():
            return b200.rewards.weighted_scores(refs, sampled, (0.7, 0.3), greedy_res=greedy, with_reward=True)
        for _ in range(3):
            call()
        torch.cuda.synchronize()
        ms = []
        for _ in range(repeats):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(launches):
                call()
            e1.record()
            e1.synchronize()
            ms.append(e0.elapsed_time(e1) / launches)
        out['weighted reward 50+10 hyps width=%d' % width] = {'ms_per_call': round(statistics.median(ms), 4), 'ms_min': round(min(ms), 4),
                                                               'ms_max': round(max(ms), 4)}
    b200.rewards.reset_scorer()
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--steps', type=int, default=3)
    p.add_argument('--repeats', type=int, default=3)
    p.add_argument('--launches', type=int, default=50)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('long_caption_rate.py measures on a CUDA device; none is visible')
    out = {'images': B, 'samples_per_image': N_PER, 'regions': R, 'steps_per_window': a.steps, 'windows': a.repeats}
    out['reward'] = reward_table(a.launches, a.repeats)
    out['decode'] = decode_table(a.steps, a.repeats)
    out['scst'] = scst_table(a.steps, a.repeats)
    out.update(device_info())
    print(json.dumps(out))


if __name__ == '__main__':
    main()
