"""GPU: the beam loop's per-step tail after the logit GEMM, kernel by kernel, with the idle gaps between them (torch.profiler trace).

    python tools/beam_loop_gaps.py [B] [beam]

UpDown, the bench.py shape (36 x 2048 features, T 20, V + 1 = 9488), three warm decodes traced.  For every step t >= 1 it reads, in
stream order, the logit GEMM, the kernels that follow it up to the next step's first GEMM, and the gaps between them; it prints the
median of each over all traced steps, and the card's name and power limit.
"""
import json
import os
import statistics
import sys
import tempfile

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from imagecaptioning.pytorch_b200 import synthetic as syn      # noqa: E402
import bench                                                    # noqa: E402

B = int(sys.argv[1]) if len(sys.argv) > 1 else 256
beam = int(sys.argv[2]) if len(sys.argv) > 2 else 5


def card():
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
        return '%s, power limit %.0f W' % (pynvml.nvmlDeviceGetName(h), pynvml.nvmlDeviceGetPowerManagementLimit(h) / 1e3)
    except Exception as e:          # the name alone when NVML is not there
        return '%s (power limit not read: %s)' % (torch.cuda.get_device_name(), e)


model = syn.build_model('updown', seed=1234, logit_scale=12.0, mode='tc_f16x3', **bench.CFG)
fc, att = syn.make_inputs(B, bench.R, 2048, 2048, seed=1)
fc, att = fc.cuda(), att.cuda()
opt = {'beam_size': beam, 'sample_n': 1}
with torch.no_grad():
    for _ in range(3):
        model(fc, att, None, opt=opt, mode='sample')
    torch.cuda.synchronize()
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            model(fc, att, None, opt=opt, mode='sample')
        torch.cuda.synchronize()
with tempfile.TemporaryDirectory() as tmp:
    path = os.path.join(tmp, 'trace.json')
    prof.export_chrome_trace(path)
    events = json.load(open(path))['traceEvents']
kern = sorted((e for e in events if e.get('cat') == 'kernel'), key=lambda e: e['ts'])


def short(name):
    for key in ('gemm_tc256_kernel', 'gemm_tc_kernel', 'vocab_stats_online128_kernel', 'beam_step_kernel', 'beam_search_step_kernel',
                'state_gather_embed_kernel'):
        if key in name:
            return key
    return name.split('(')[0][-48:]


STEP_KERNELS = ('vocab_stats_online128_kernel', 'beam_step_kernel', 'state_gather_embed_kernel', 'beam_search_step_kernel')
# a step's tail: from the logit GEMM (the GEMM right before the vocabulary kernel) to the next step's first GEMM
tails = []
for i, e in enumerate(kern):
    n = short(e['name'])
    if n not in ('vocab_stats_online128_kernel', 'beam_search_step_kernel'):
        continue
    j = i
    while j + 1 < len(kern) and not short(kern[j + 1]['name']).startswith('gemm_tc'):
        j += 1
    if j + 1 >= len(kern) or i == 0:
        continue
    seq = kern[i - 1:j + 2]                   # logit GEMM, tail kernels, next GEMM
    if not all(short(k['name']) in STEP_KERNELS for k in seq[1:-1]):
        continue                              # the last step: beam finalize, the log-prob gather and the next decode's prologue follow
    tails.append(seq)
T = bench.CFG['T']
if len(tails) != 3 * (T - 1):
    sys.exit('expected %d step tails (steps 0 .. T-2 of three decodes), found %d' % (3 * (T - 1), len(tails)))
tails = [s for i, s in enumerate(tails) if i % (T - 1) != 0]       # step 0 runs B rows, not B * beam
shape = [short(k['name']) for k in tails[0][1:-1]]
tails = [s for s in tails if [short(k['name']) for k in s[1:-1]] == shape]
print('%s; UpDown B=%d beam=%d, %d steps t >= 1 traced (medians, us)' % (card(), B, beam, len(tails)))
total = []
for s in tails:
    total.append(s[-1]['ts'] - (s[0]['ts'] + s[0]['dur']))
prev = 'logit GEMM'
for p in range(1, len(shape) + 1):
    gap = statistics.median(s[p]['ts'] - (s[p - 1]['ts'] + s[p - 1]['dur']) for s in tails)
    dur = statistics.median(s[p]['dur'] for s in tails)
    print('  gap %-30s -> %-30s %7.2f' % (prev, shape[p - 1], gap))
    print('  %-67s %7.2f' % (shape[p - 1], dur))
    prev = shape[p - 1]
gap = statistics.median(s[-1]['ts'] - (s[-2]['ts'] + s[-2]['dur']) for s in tails)
print('  gap %-30s -> %-30s %7.2f' % (prev, 'next step GEMM', gap))
print('  logit GEMM end -> next step GEMM start: %.2f us per step' % statistics.median(total))
