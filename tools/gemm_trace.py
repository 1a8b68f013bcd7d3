"""GPU: where the time of one decode GEMM launch goes.  Runs the 3-pass wgmma kernel on a decode-step shape with the phase stamps on
(capb200_gemm_trace) and prints, relative to the earliest set-up stamp, when each phase happened (median / max over the CTAs).

    python tools/gemm_trace.py [M N K]        default: the language-LSTM gates of the headline shape, 1280 x 4000 x 3000
"""
import os, sys
import numpy as np
import torch
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import imagecaptioning.pytorch_b200 as b200
L = b200._lib
lib = L.load()
M, N, K = (int(v) for v in sys.argv[1:4]) if len(sys.argv) >= 4 else (1280, 4000, 3000)
x = torch.randn(M, K, device='cuda'); w = torch.randn(N, K, device='cuda') / K ** 0.5; y = torch.empty(M, N, device='cuda')
tr = np.zeros((296, 16), dtype=np.uint64)
L.check(lib.capb200_gemm_trace(L.ptr(x), L.ptr(w), L.ptr(y), M, N, K, tr.ctypes.data, tr.size, L.current_stream()), 'gemm_trace')
used = tr[:, 0] > 0
t = tr[used].astype(np.float64)
t0 = t[:, 0].min()
names = ['set-up done', 'first operands landed', 'tile 0: main loop done', 'tile 1: main loop done', '(unused)', '(unused)',
         'tile 0: epilogue done', 'tile 1: epilogue done', 'kernel end']
print('decode GEMM %d x %d x %d, %d CTAs traced; times in us after the first CTA finished its set-up' % (M, N, K, int(used.sum())))
for i, n in enumerate(names):
    col = t[:, i]
    col = col[col > 0]
    if col.size == 0:
        continue
    print('%-34s  n=%3d  min %7.2f  median %7.2f  max %7.2f' % (n, col.size, (col.min() - t0) / 1e3, (np.median(col) - t0) / 1e3, (col.max() - t0) / 1e3))
lead = t[(t[:, 2] > 0)]
if lead.size:
    d01 = (lead[:, 2] - lead[:, 1]) / 1e3
    print('first operands -> tile 0 main loop done: median %.2f us (%d K-blocks => %.3f us per K-block)' % (np.median(d01), -(-K // 64), np.median(d01) / (-(-K // 64))))
    two = lead[lead[:, 3] > 0]
    if two.size:
        d12 = (two[:, 3] - two[:, 2]) / 1e3
        print('CTAs with two tiles: tile 0 main loop -> tile 1 main loop: median %.2f us' % np.median(d12))
