"""GPU: the decode GEMM's ping-pong schedule (consumer warpgroup 1 runs a CTA's even tiles, warpgroup 2 its odd ones, their main loops
taking turns) at tile counts per CTA of one, one or two, an odd count (SM count + 1 tiles) and five or six, with K-blocks per tile both
below and above the ring depth.  Every epilogue kind is checked against float64, the LSTM kind with fresh (src_row = -1) and permuted
source rows, and a second launch of the same problem must give bitwise the same outputs."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

EPS_FAST = 1e-6   # fast_sigmoid / fast_tanh absolute error (common.cuh), as in test_gpu_decode_gemm_epilogue.py


def _shape(name):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return {'one_tile': (256, 4000, 200),           # 64-wide tiles, fewer than the SMs: one tile per CTA (the t = 0 gate shape)
            'two_tiles': (1280, 4000, 200),         # 160-wide: 250 tiles, one or two per CTA
            'sms_plus_one': (128 * (sms + 1), 64, 64),   # one K-block; CTA 0 runs two tiles, the rest one
            'five_six': (1280, 9488, 128)}[name]    # 750 tiles: five or six per CTA, two K-blocks per tile


@pytest.fixture(scope='module')
def L():
    import imagecaptioning.pytorch_b200 as b200
    return b200._lib


def _run(L, lib, x, w, M, N, K, epi):
    L.check(lib.capb200_decode_gemm(L.ptr(x), L.ptr(w), M, N, K, L.OP_MODES['tc_f16x3'], epi, None, 0, L.current_stream()), 'decode_gemm')
    torch.cuda.synchronize()


@pytest.mark.parametrize('kind', ['store', 'planes', 'lstm_permuted', 'lstm_identity'])
@pytest.mark.parametrize('name', ['one_tile', 'two_tiles', 'sms_plus_one', 'five_six'])
def test_pingpong_matches_fp64_and_repeats(L, name, kind):
    M, N, K = _shape(name)
    lib = L.load()
    g = torch.Generator().manual_seed(M + N + K)
    x = torch.randn(M, K, generator=g)
    w = (torch.rand(N, K, generator=g) * 2 - 1) / K ** 0.5
    b = torch.randn(N, generator=g)
    xd, wd, bd = x.cuda(), w.cuda(), b.cuda()
    z64 = (x.double() @ w.double().t() + b.double()).numpy()
    err32 = float(np.abs((x @ w.t() + b).double().numpy() - z64).max())
    tol = max(4 * err32, 2e-6) + 3 * (K / 16) * 2.0 ** -24 * float(np.abs(z64).max())
    epi = L.GemmEpilogue()
    epi.bias = L.ptr(bd)

    if kind in ('store', 'planes'):
        y = torch.full((M, N), float('nan'), device='cuda')
        planes = torch.zeros(2, M, N, dtype=torch.float16, device='cuda')
        epi.C, epi.ldc = L.ptr(y), N
        if kind == 'planes':
            epi.C_hi, epi.C_lo, epi.ldcs = L.ptr(planes[0]), L.ptr(planes[1]), N
        _run(L, lib, xd, wd, M, N, K, epi)
        first = (y.clone(), planes.clone())
        err = float(np.abs(y.cpu().double().numpy() - z64).max())
        assert err < tol, (name, kind, err, tol)
        if kind == 'planes':
            assert torch.equal(planes[0], y.half()) and torch.equal(planes[1], (y - planes[0].float()).half())
        _run(L, lib, xd, wd, M, N, K, epi)
        assert torch.equal(first[0], y) and torch.equal(first[1], planes)
        return

    H = N // 4
    c_prev = torch.randn(M, H, generator=g)
    if kind == 'lstm_permuted':
        srow = torch.randperm(M, generator=g).int()
        srow[::5] = -1                                                   # fresh rows start from the zero state
        srow_d = srow.cuda()
        epi.src_row = L.ptr(srow_d)
        cp = torch.where((srow >= 0)[:, None], c_prev[srow.long().clamp_min(0)], torch.zeros(()))
    else:
        cp = c_prev
    cp = cp.double().numpy()
    cprev_d = c_prev.cuda()
    c_out = torch.full((M, H), float('nan'), device='cuda')
    h_f = torch.full((M, H), float('nan'), device='cuda')
    hp = torch.zeros(2, M, H, dtype=torch.float16, device='cuda')
    epi.lstm, epi.H = 1, H
    epi.c_prev, epi.ld_cprev = L.ptr(cprev_d), H
    epi.c_out, epi.ld_cout = L.ptr(c_out), H
    epi.h_f, epi.ld_h = L.ptr(h_f), H
    epi.h_hi, epi.h_lo = L.ptr(hp[0]), L.ptr(hp[1])
    _run(L, lib, xd, wd, M, N, K, epi)
    sig = lambda v: 1.0 / (1.0 + np.exp(-v))
    zi, zf, zg, zo = (z64[:, q::4] for q in range(4))
    c_ref = sig(zf) * cp + sig(zi) * np.tanh(zg)
    h_ref = sig(zo) * np.tanh(c_ref)
    cmax = float(np.abs(cp).max())
    tol_c = (tol / 4 + EPS_FAST) * cmax + (tol / 4 + EPS_FAST) + (tol + EPS_FAST)
    tol_h = (tol / 4 + EPS_FAST) + tol_c + EPS_FAST
    err_c = float(np.abs(c_out.cpu().double().numpy() - c_ref).max())
    err_h = float(np.abs(h_f.cpu().double().numpy() - h_ref).max())
    assert err_c < tol_c and err_h < tol_h, (name, kind, err_c, tol_c, err_h, tol_h)
    assert torch.equal(hp[0], h_f.half()) and torch.equal(hp[1], (h_f - hp[0].float()).half())
    first = (c_out.clone(), h_f.clone(), hp.clone())
    _run(L, lib, xd, wd, M, N, K, epi)
    assert torch.equal(first[0], c_out) and torch.equal(first[1], h_f) and torch.equal(first[2], hp)
