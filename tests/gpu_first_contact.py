"""Stand-alone first-contact script for a fresh GPU machine: exercises the wgmma GEMM on a few shapes with a hard
process-level timeout around each launch group, so a protocol bug becomes a log line rather than a hung box.
Usage: python tests/gpu_first_contact.py   (writes to stdout)"""
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import __graft_entry__ as ge   # noqa: E402

ge.build()
import imagecaptioning.pytorch_b200 as b200   # noqa: E402

L = b200._lib
lib = L.load()
print('device', torch.cuda.get_device_name(0), 'cc', torch.cuda.get_device_capability(0))


def run(M, N, K, mode, relu=False):
    g = torch.Generator().manual_seed(M + N + K)
    x = torch.randn(M, K, generator=g)
    w = (torch.rand(N, K, generator=g) * 2 - 1) / K ** 0.5
    b = torch.randn(N, generator=g)
    ref = x.double() @ w.double().t() + b.double()
    xd, wd, bd = x.cuda(), w.cuda(), b.cuda()
    y = torch.full((M, N), float('nan'), device='cuda')
    rc = lib.capb200_linear(L.ptr(xd), K, L.ptr(wd), K, L.ptr(bd), L.ptr(y), N, M, N, K, int(relu), L.MODES[mode], L.current_stream())
    torch.cuda.synchronize()
    err = float((y.cpu().double() - ref).abs().max())
    fp32 = float(((x @ w.t() + b).double() - ref).abs().max())
    print('linear %-10s M=%5d N=%5d K=%5d rc=%d max|err|=%.3e (torch fp32: %.3e) nan=%d' % (mode, M, N, K, rc, err, fp32, int(torch.isnan(y).sum())), flush=True)
    return err


for mode in ('simt_fp32', 'tc_f16x1', 'tc_f16x3'):
    for (M, N, K) in [(128, 128, 64), (128, 128, 256), (256, 256, 1000), (130, 260, 1000), (1280, 4000, 1000), (77, 9488, 1000)]:
        run(M, N, K, mode)

# timing of the headline GEMM shapes
for mode in ('simt_fp32', 'tc_f16x1', 'tc_f16x3'):
    for (M, N, K) in [(1280, 4000, 3000), (1280, 9488, 1000), (9216, 1000, 2048)]:
        x = torch.randn(M, K, device='cuda'); w = torch.randn(N, K, device='cuda') / K ** 0.5; b = torch.randn(N, device='cuda')
        y = torch.empty(M, N, device='cuda')
        # note: capb200_linear re-splits operands every call in the tensor-core modes, so this is an upper bound
        for _ in range(2):
            lib.capb200_linear(L.ptr(x), K, L.ptr(w), K, L.ptr(b), L.ptr(y), N, M, N, K, 0, L.MODES[mode], L.current_stream())
        torch.cuda.synchronize()
        t0 = time.time()
        for _ in range(5):
            lib.capb200_linear(L.ptr(x), K, L.ptr(w), K, L.ptr(b), L.ptr(y), N, M, N, K, 0, L.MODES[mode], L.current_stream())
        torch.cuda.synchronize()
        dt = (time.time() - t0) / 5
        print('time %-10s M=%5d N=%5d K=%5d  %.3f ms  %.1f TFLOP/s (incl. operand split)' % (mode, M, N, K, dt * 1e3, 2.0 * M * N * K / dt / 1e12), flush=True)
print('first contact done')
