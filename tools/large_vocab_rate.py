"""Cost of vocabularies above 51 199 words.

1. The vocabulary step alone (capb200_vocab_select: log-softmax of each row in place plus the word choice) for greedy, multinomial,
   top-5 and top-0.9 at V + 1 = 51 200 (the last length one CTA caches: vocab_step_kernel) and 51 201 / 100 001 / 409 600 (the
   thread-block cluster form, 2 / 2 / 8 CTAs per row), with 1, 50 and 1280 rows.  CUDA events around `--launches` launches.
2. UpDown end to end at V = 9487 against V = 100 000 (E = H = 1000, A = 512, 36 regions, T = 16, tc_f16x3): a greedy decode of 50
   images, and the fused self-critical step of 10 images x 5 samples (graph replays, as training runs it).

Prints one JSON line with the card name and power limit read in the same run.

    python tools/large_vocab_rate.py [--launches 200] [--repeats 5] [--steps 10] [--skip-model]
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tools'))

from dbs_rate import device_info      # noqa: E402

SELECTS = {'greedy': (1, 0.0), 'sample': (2, 0.0), 'top5': (4, 5.0), 'top0.9': (5, 0.9)}
LENGTHS = [51200, 51201, 100001, 409600]
ROWS = [1, 50, 1280]


def vocab_step_ms(L, V1, rows, select, top, launches, repeats):
    """Median (min, max) over `repeats` windows of ms per launch."""
    g = torch.Generator(device='cuda').manual_seed(V1 + rows)
    x = torch.randn(rows, V1, generator=g, device='cuda') * 4
    tokens = torch.empty(rows, dtype=torch.int32, device='cuda')
    picked = torch.empty(rows, device='cuda')
    lib, st = L.load(), L.current_stream()

    def launch(i):
        # the row is rewritten with its log-softmax, a fixed point of the step: every launch sees the same distribution
        L.check(lib.capb200_vocab_select(L.ptr(x), V1, rows, V1, select, top, 1.0, 7, i, None, 1, L.ptr(tokens), L.ptr(picked), st), 'vocab_select')

    for i in range(10):
        launch(i)
    torch.cuda.synchronize()
    ms = []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(launches):
            launch(i)
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1) / launches)
    return {'ms': round(statistics.median(ms), 4), 'min': round(min(ms), 4), 'max': round(max(ms), 4)}


def vocab_step_table(L, launches, repeats, lengths=LENGTHS, rows_list=ROWS):
    out = {}
    for V1 in lengths:
        for rows in rows_list:
            for name, (select, top) in SELECTS.items():
                out['V1=%d rows=%d %s' % (V1, rows, name)] = vocab_step_ms(L, V1, rows, select, top, launches, repeats)
    return out


def timed(step, steps, warmup, repeats):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    ms = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        for _ in range(steps):
            step()
        torch.cuda.synchronize()
        ms.append(1e3 * (time.perf_counter() - t0) / steps)
    return {'ms_per_call': round(statistics.median(ms), 3), 'ms_min': round(min(ms), 3), 'ms_max': round(max(ms), 3)}


def updown_table(steps, repeats):
    from imagecaptioning.pytorch_b200 import rewards
    from imagecaptioning.pytorch_b200 import synthetic as syn
    out = {}
    R, T = 36, 16
    for V in (9487, 100000):
        cfg = dict(V=V, E=1000, H=1000, A=512, F_fc=2048, F_att=2048, T=T)
        model = syn.build_model('updown', seed=1234, logit_scale=6.0, mode='tc_f16x3', device=torch.device('cuda:0'), heads=8, **cfg)
        fc, att = syn.make_inputs(50, R, cfg['F_fc'], cfg['F_att'], seed=1234)
        fc, att = fc.cuda(), att.cuda()

        def decode():
            with torch.no_grad():
                model(fc, att, None, opt={'sample_method': 'greedy', 'beam_size': 1}, mode='sample')

        model.eval()
        res = {'greedy_decode_50_images': timed(decode, steps, 3, repeats)}
        model.train()
        refs = syn.make_refs(200, V, seed=4)
        table = rewards.CiderDTable(*syn.document_frequency(refs))
        res['scst_step_10x5'] = timed(lambda: model.scst_step(fc[:10], att[:10], refs[:10], table, 5), steps, 3, repeats)
        out['V=%d' % V] = res
        del model
        torch.cuda.empty_cache()
    for k in ('greedy_decode_50_images', 'scst_step_10x5'):
        out['V=100000 over V=9487 ' + k] = round(out['V=100000'][k]['ms_per_call'] / out['V=9487'][k]['ms_per_call'], 3)
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--launches', type=int, default=200)
    p.add_argument('--repeats', type=int, default=5)
    p.add_argument('--steps', type=int, default=10)
    p.add_argument('--skip-model', action='store_true')
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('large_vocab_rate.py measures on a CUDA device; none is visible')
    import imagecaptioning.pytorch_b200 as b200
    out = {'launches_per_window': a.launches, 'windows': a.repeats}
    out['vocab_step_ms_per_launch'] = vocab_step_table(b200._lib, a.launches, a.repeats)
    if not a.skip_model:
        out['updown'] = updown_table(a.steps, a.repeats)
    out.update(device_info())
    print(json.dumps(out))


if __name__ == '__main__':
    main()
