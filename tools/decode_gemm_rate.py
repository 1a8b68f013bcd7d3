"""GPU: time the decode GEMM (tc_f16x3) at the shapes of the UpDown decode step (beam 5, batch 256: 1280 rows) and its prologue under
both schedules (gemm_tc_kernel, 128-row tiles; gemm_tc256_kernel, 256-row tiles), with the tile height the launch rule picks and
torch.matmul in fp16 at the same M x N x K beside each row as this card's practical one-pass tensor rate.  TFLOP/s are algorithmic
(2 M N K per launch, not counting the three passes).

    python tools/decode_gemm_rate.py [iters]
"""
import os, sys, subprocess
import torch
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import imagecaptioning.pytorch_b200 as b200
L = b200._lib
lib = L.load()
iters = int(sys.argv[1]) if len(sys.argv) > 1 else 200
# The step at t = 0 launches the 1280-row gate plans with M = 256, so it runs with the tile width of the 1280-row shape.
SHAPES = [('lang_lstm gates', 1280, 4000, 3000), ('att_lstm gates', 1280, 4000, 2000), ('logit', 1280, 9488, 1000), ('h2att', 1280, 512, 1000),
          ('att_embed', 9216, 1000, 2048), ('ctx2att', 9216, 512, 1000)]


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30)
        return q.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + ' (power limit not readable)'


def torch_ms(a, b):
    for _ in range(3):
        torch.matmul(a, b.t())
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        torch.matmul(a, b.t())
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def f16x3_ms(x, w, b, y, M, N, K, bm):
    # CAPB200_GEMM_BM is read at every launch: 128 forces the ping-pong schedule, 256 the cooperative one (where BN has it), None the rule
    if bm is None:
        os.environ.pop('CAPB200_GEMM_BM', None)
    else:
        os.environ['CAPB200_GEMM_BM'] = str(bm)
    ms = torch.zeros(1)
    L.check(lib.capb200_bench_linear(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(y), M, N, K, L.OP_MODES['tc_f16x3'], iters, ms.numpy().ctypes.data,
                                     L.current_stream()), 'bench_linear')
    os.environ.pop('CAPB200_GEMM_BM', None)
    return float(ms[0])


print('card: %s' % card())
print('f16x3 ms under each schedule: BM 128 (ping-pong, 128 x BN tiles) and BM 256 (cooperative, 256 x BN tiles; BN 64 has none); '
      'BM is the rule\'s choice')
print('%-22s %5s %5s %5s %4s %4s  %9s %8s  %9s %8s  %12s %10s' % ('GEMM', 'M', 'N', 'K', 'BN', 'BM', 'BM128 ms', 'TFLOP/s', 'BM256 ms', 'TFLOP/s',
                                                               'torch f16 ms', 'TFLOP/s'))
g = torch.Generator(device='cuda').manual_seed(0)
for name, M, N, K in SHAPES:
    x = torch.randn(M, K, device='cuda', generator=g); w = torch.randn(N, K, device='cuda', generator=g) / K ** 0.5
    b = torch.zeros(N, device='cuda'); y = torch.empty(M, N, device='cuda')
    bn = lib.capb200_gemm_tile_n(M, N)
    ms128 = f16x3_ms(x, w, b, y, M, N, K, 128)
    ms256 = f16x3_ms(x, w, b, y, M, N, K, 256) if bn != 64 else float('nan')
    t_ms = torch_ms(x.half(), w.half())
    flop = 2.0 * M * N * K
    print('%-22s %5d %5d %5d %4d %4d  %9.4f %8.1f  %9.4f %8.1f  %12.4f %10.1f' % (name, M, N, K, bn, lib.capb200_gemm_tile_m(M, N), ms128, flop / ms128 / 1e9,
                                                                              ms256, flop / ms256 / 1e9, t_ms, flop / t_ms / 1e9))
