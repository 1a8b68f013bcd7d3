"""GPU: time the training-step GEMM shapes of BASELINE configs[3] (AoANet, 10 images x 5 samples) on the wgmma tf32 kernel and on the
mma.sync kernel it replaced; reports microseconds per launch and the fraction of the HBM roofline (fp32 weight bytes / time).

    python tools/tf32_sweep.py [iters]
"""
import json, os, sys
import torch
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import imagecaptioning.pytorch_b200 as b200
L = b200._lib
lib = L.load()
iters = int(sys.argv[1]) if len(sys.argv) > 1 else 50
peaks = os.path.join(REPO, 'MEASURED_PEAKS.json')
hbm = json.load(open(peaks))['hbm_gbs'] if os.path.exists(peaks) else 6650.0
SHAPES = [('att_lstm gates (3 segments in the step)', 50, 4096, 3072), ('attention q-projection', 50, 1024, 1024), ('att2ctx', 50, 2048, 2048),
          ('logit', 50, 9488, 1024), ('d gates -> d x (W^T)', 50, 1024, 4096), ('refiner q|k|v', 360, 3072, 1024), ('refiner AoA', 360, 2048, 2048),
          ('logit input gradient, batched over time', 1000, 1024, 9488), ('weight gradient att_lstm (out x in over T*N rows)', 4096, 1024, 1000),
          ('weight gradient logit', 9488, 1024, 1000), ('greedy-sized rows', 10, 4096, 3072)]
print('%-52s %6s %6s %6s  %10s %10s  %8s %8s' % ('call site', 'M', 'N', 'K', 'wgmma us', 'mma.sync us', 'GB/s', 'of HBM'))
for name, M, N, K in SHAPES:
    x = torch.randn(M, K, device='cuda'); w = torch.randn(N, K, device='cuda') / K ** 0.5; b = torch.zeros(N, device='cuda'); y = torch.empty(M, N, device='cuda')
    out = []
    for mode in ('tf32x3_tc', 'skinny_tf32x3'):
        ms = torch.zeros(1, dtype=torch.float32)
        # rotate nothing: weights of one call site (<= 50 MB) would sit in L2 across back-to-back launches, so flush L2 between timings is
        # NOT done here; the step itself streams ~110 MB of weights per time step, see the in-step numbers of tools/scst_table.py
        L.check(lib.capb200_bench_linear(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y), M, N, K, L.OP_MODES[mode], iters, ms.numpy().ctypes.data, L.current_stream()), 'bench_linear')
        out.append(float(ms[0]) * 1e3)
    bytes_ = 4.0 * (N * K + M * K + M * N)
    gbs = bytes_ / (out[0] * 1e-6) / 1e9
    print('%-52s %6d %6d %6d  %10.1f %10.1f  %8.0f %8.2f' % (name, M, N, K, out[0], out[1], gbs, gbs / hbm))
