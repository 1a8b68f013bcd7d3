"""GPU: where the time of one decode GEMM launch goes.  Runs the 3-pass wgmma kernel on a decode-step shape with the phase stamps on
(capb200_decode_gemm with a trace buffer) and prints, relative to the earliest set-up stamp, when each phase happened (median / max over
the CTAs), the epilogue time per tile and whether tile 0's epilogue (consumer warpgroup 1) ended before tile 1's main loop (warpgroup 2)
did.  With --epilogue lstm it also splits the first 64 rows of each tile's LSTM epilogue into bias adds and c_prev loads, cell math, and
stores.

    python tools/gemm_trace.py [--epilogue store|planes|lstm] [M N K]

default shape: the language-LSTM gates of the headline shape, 1280 x 4000 x 3000.  Epilogues as the decode step runs them:
    store    fp32 C + bias (logit, h2att, ctx2att)
    planes   fp32 C + split fp16 planes + bias + ReLU (fc_embed, att_embed)
    lstm     fused LSTM cell: bias, c_prev read through a permuted src_row, c_out, h and its split planes (language LSTM, N = 4H)
"""
import argparse, os, sys
import numpy as np
import torch
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import imagecaptioning.pytorch_b200 as b200
L = b200._lib
lib = L.load()
ap = argparse.ArgumentParser()
ap.add_argument('--epilogue', choices=['store', 'planes', 'lstm'], default='store')
ap.add_argument('shape', nargs='*', type=int, default=[1280, 4000, 3000])
args = ap.parse_args()
M, N, K = args.shape
x = torch.randn(M, K, device='cuda'); w = torch.randn(N, K, device='cuda') / K ** 0.5
epi = L.GemmEpilogue()
bias = torch.randn(N, device='cuda')
epi.bias = L.ptr(bias)
keep = [bias]
if args.epilogue == 'lstm':
    H = N // 4
    c_prev = torch.randn(M, H, device='cuda'); c_out = torch.empty(M, H, device='cuda'); h = torch.empty(M, H, device='cuda')
    hp = torch.empty(2, M, H, dtype=torch.float16, device='cuda')
    src = torch.randperm(M, device='cuda').int()
    keep += [c_prev, c_out, h, hp, src]
    epi.lstm, epi.H = 1, H
    epi.c_prev, epi.ld_cprev, epi.src_row = L.ptr(c_prev), H, L.ptr(src)
    epi.c_out, epi.ld_cout = L.ptr(c_out), H
    epi.h_f, epi.h_hi, epi.h_lo, epi.ld_h = L.ptr(h), L.ptr(hp[0]), L.ptr(hp[1]), H
else:
    y = torch.empty(M, N, device='cuda')
    keep.append(y)
    epi.C, epi.ldc = L.ptr(y), N
    if args.epilogue == 'planes':
        yp = torch.empty(2, M, N, dtype=torch.float16, device='cuda')
        keep.append(yp)
        epi.C_hi, epi.C_lo, epi.ldcs, epi.relu = L.ptr(yp[0]), L.ptr(yp[1]), N, 1
tr = np.zeros((296, 16), dtype=np.uint64)
L.check(lib.capb200_decode_gemm(L.ptr(x), L.ptr(w), M, N, K, L.OP_MODES['tc_f16x3'], epi, tr.ctypes.data, tr.size, L.current_stream()),
        'decode_gemm')
used = tr[:, 0] > 0
t = tr[used].astype(np.float64)
t0 = t[:, 0].min()
BM = lib.capb200_gemm_tile_m(M, N)    # CAPB200_GEMM_BM=128 / 256 picks the schedule to trace
if BM == 128:   # ping-pong: warpgroup 1 runs tile 0, warpgroup 2 tile 1
    part = ['tile 0', 'tile 1']
    names = ['set-up done', 'first operands landed', 'tile 0: main loop done', 'tile 1: main loop done', 'tile 1: main loop starts', '(unused)',
             'tile 0: epilogue done', 'tile 1: epilogue done', 'kernel end']
else:           # cooperative: both warpgroups run rows 0..127 / 128..255 of tile 0
    part = ['warpgroup 1', 'warpgroup 2']
    names = ['set-up done', 'first operands landed', 'warpgroup 1: tile 0 main loop done', 'warpgroup 2: tile 0 main loop done', '(unused)',
             'producer: tile 0 last K-block issued', 'warpgroup 1: tile 0 epilogue done', 'warpgroup 2: tile 0 epilogue done', 'kernel end']
names += ['%s lstm: %s' % (w, s) for w in part for s in ('c_prev landed', 'cell math done', 'stores issued')]
print('decode GEMM %d x %d x %d, %s epilogue, BM %d, BN %d, %d CTAs traced; times in us after the first CTA finished its set-up'
      % (M, N, K, args.epilogue, BM, lib.capb200_gemm_tile_n(M, N), int(used.sum())))
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
    epi0 = (lead[:, 6] - lead[:, 2]) / 1e3
    print('epilogue of tile 0: median %.2f us, max %.2f us' % (np.median(epi0), epi0.max()))
    two = lead[lead[:, 3] > 0]
    if two.size and BM == 128:
        d12 = (two[:, 3] - two[:, 2]) / 1e3
        epi1 = (two[:, 7] - two[:, 3]) / 1e3
        print('CTAs with two tiles: tile 0 main loop -> tile 1 main loop: median %.2f us; epilogue of tile 1: median %.2f us, max %.2f us'
              % (np.median(d12), np.median(epi1), epi1.max()))
        hidden = two[:, 6] <= two[:, 3]
        print('tile 0 epilogue ended before tile 1 main loop did: %d of %d CTAs' % (int(hidden.sum()), len(two)))
    if args.epilogue == 'lstm':
        for who, (done, first) in zip(part, [(2, 9), (3, 12)]):
            r = lead[(lead[:, done] > 0) & (lead[:, first + 2] > 0)]
            if r.size == 0:
                continue
            parts = [(r[:, first] - r[:, done]) / 1e3, (r[:, first + 1] - r[:, first]) / 1e3, (r[:, first + 2] - r[:, first + 1]) / 1e3]
            print('%s lstm epilogue, its first 64 rows, median (max) us: adds + c_prev loads %.2f (%.2f), cell math %.2f (%.2f), stores %.2f (%.2f)'
                  % ((who,) + tuple(v for q in parts for v in (np.median(q), q.max()))))
