"""GPU: every epilogue kind of the decode GEMM (fp32 store, store + split planes, fused LSTM cell) at every tile width (64, 128, 160
columns), through capb200_decode_gemm, against a float64 reference.  M and N are ragged against the 128-row and BN-column tiles, K against
the 64-wide K-block, and every launch-wide option is exercised: bias, row bias with rows_per_group 5, gathered bias with repeated tokens,
residual, ReLU, src_row with -1 (zero state) and a permutation, unaligned output pitches, and split planes that must reconstruct the
fp32 output."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# (M, N, K) and the tile width a 132-SM H100 SXM picks for it; N is a multiple of 4 so the same shapes serve the LSTM kind (H = N / 4)
SHAPES = [(130, 1000, 200, 64), (1205, 9488, 200, 128), (1205, 4040, 200, 160)]
CASES = [
    # kind, options
    ('store', dict(bias=True)),
    ('store', dict(bias=True, relu=True, residual=True, odd_pitch=True)),
    ('planes', dict(bias=True, relu=True)),
    ('planes', dict(bias=True, no_c=True, odd_pitch=True)),
    ('lstm', dict(row_bias=True, gather=True, src='permuted', planes=True)),      # attention LSTM of the decode step
    ('lstm', dict(bias=True, residual=True, src='identity')),                     # language LSTM after the split gate sum
    ('lstm', dict(bias=True, src='permuted', no_cprev=True, odd_pitch=True)),
]
EPS_FAST = 1e-6   # fast_sigmoid / fast_tanh: absolute error < 3e-7 (common.cuh), with room for the rounding of the cell's products


@pytest.fixture(scope='module')
def L():
    import imagecaptioning.pytorch_b200 as b200
    return b200._lib


def test_shapes_cover_every_tile_width(L):
    if torch.cuda.get_device_properties(0).multi_processor_count != 132:
        pytest.skip('the widths noted in SHAPES are those of a 132-SM H100 SXM; the choice follows the SM count')
    lib = L.load()
    assert [lib.capb200_gemm_tile_n(M, N) for M, N, _, _ in SHAPES] == [bn for _, _, _, bn in SHAPES]


def _linear_tol(err32, ref, K):
    # the bar of test_gpu_decode_gemm.py: summation-order noise of fp32 plus one fp32 ulp of the largest output per accumulate
    return max(4 * err32, 2e-6) + 3 * (K / 16) * 2.0 ** -24 * float(np.abs(ref).max())


def _check_planes(hi, lo, full):
    # split_f32: hi = fp16(x), lo = fp16(x - hi); x - hi is exact in fp32, so both planes are determined bit for bit by the fp32 value
    assert torch.equal(hi, full.half())
    assert torch.equal(lo, (full - hi.float()).half())


@pytest.mark.parametrize('shape', SHAPES, ids=lambda s: 'M%d_N%d_K%d_bn%d' % s)
@pytest.mark.parametrize('kind,opt', CASES, ids=['%s%d' % (k, i) for i, (k, _) in enumerate(CASES)])
def test_epilogue_matches_fp64(L, shape, kind, opt):
    M, N, K, _ = shape
    lib = L.load()
    g = torch.Generator().manual_seed(M + 3 * N + K + len(opt))
    x = torch.randn(M, K, generator=g)
    w = (torch.rand(N, K, generator=g) * 2 - 1) / K ** 0.5
    xd, wd = x.cuda(), w.cuda()      # held until the call returns: a freed temporary's memory can be handed to the next one
    epi = L.GemmEpilogue()
    keep = []

    def dev(t):
        t = t.cuda()
        keep.append(t)
        return L.ptr(t)

    # pre-activation in float64 and in fp32 (the latter only sizes the summation-order noise of the bar)
    z64 = x.double() @ w.double().t()
    z32 = x @ w.t()
    if opt.get('bias'):
        b = torch.randn(N, generator=g)
        epi.bias = dev(b)
        z64 += b.double(); z32 += b
    if opt.get('row_bias'):
        G = -(-M // 5)
        rb = torch.randn(G, N + 3, generator=g)
        epi.row_bias, epi.ld_row_bias, epi.rows_per_group = dev(rb), N + 3, 5
        rows = torch.arange(M) // 5
        z64 += rb[rows, :N].double(); z32 += rb[rows, :N]
    if opt.get('gather'):
        tab = torch.randn(7, N + 5, generator=g)
        idx = torch.randint(0, 7, (M,), generator=g, dtype=torch.int32)   # 7 tokens over M rows: repeated
        epi.gather_bias, epi.ld_gb, epi.gather_idx = dev(tab), N + 5, dev(idx)
        z64 += tab[idx.long(), :N].double(); z32 += tab[idx.long(), :N]
    if opt.get('residual'):
        res = torch.randn(M, N + 1, generator=g)
        epi.residual, epi.ld_res = dev(res), N + 1
        z64 += res[:, :N].double(); z32 += res[:, :N]
    if opt.get('relu'):
        epi.relu = 1
        z64 = z64.clamp_min(0); z32 = z32.clamp_min(0)
    z64 = z64.numpy()
    tol = _linear_tol(float(np.abs(z32.double().numpy() - z64).max()), z64, K)
    pad = 1 if opt.get('odd_pitch') else 0      # an odd pitch sends odd rows down the scalar store path

    if kind in ('store', 'planes'):
        ld = N + pad
        y = torch.full((M, ld), float('nan'), device='cuda')
        planes = torch.zeros(2, M, ld, dtype=torch.float16, device='cuda')
        if not opt.get('no_c'):
            epi.C, epi.ldc = L.ptr(y), ld
        if kind == 'planes':
            epi.C_hi, epi.C_lo, epi.ldcs = L.ptr(planes[0]), L.ptr(planes[1]), ld
        L.check(lib.capb200_decode_gemm(L.ptr(xd), L.ptr(wd), M, N, K, L.OP_MODES['tc_f16x3'], epi, None, 0, L.current_stream()),
                'decode_gemm')
        torch.cuda.synchronize()
        if opt.get('no_c'):
            assert torch.isnan(y).all()
            hi, lo = planes[0, :, :N].cpu(), planes[1, :, :N].cpu()
            full = hi.double() + lo.double()
            # hi + lo carries the fp32 value to within its own 2^-22 relative plus fp16's smallest step
            err = float(np.abs(full.numpy() - z64).max())
            assert err < tol + 2.0 ** -21 * float(np.abs(z64).max()) + 2.0 ** -24, (err, tol)
            return
        out = y[:, :N].cpu()
        assert torch.isnan(y[:, N:]).all()
        err = float(np.abs(out.double().numpy() - z64).max())
        assert err < tol, (shape, kind, opt, err, tol)
        if kind == 'planes':
            _check_planes(planes[0, :, :N].cpu(), planes[1, :, :N].cpu(), out)
        return

    # fused LSTM cell; gate columns are interleaved: column 4u + q holds gate q in (i, f, g, o) of unit u
    H = N // 4
    ldc = H + pad
    c_prev = torch.randn(M + 3, ldc, generator=g)
    src = opt.get('src')
    if src == 'permuted':
        srow = torch.randperm(M, generator=g).int()
        srow[::7] = -1                                                   # fresh rows start from the zero state
        epi.src_row = dev(srow)
        src_idx = srow.long()
    else:
        src_idx = torch.arange(M)
    if not opt.get('no_cprev'):
        epi.c_prev, epi.ld_cprev = dev(c_prev), ldc
        cp = torch.where((src_idx >= 0)[:, None], c_prev[src_idx.clamp_min(0), :H], torch.zeros(()))
    else:
        cp = torch.zeros(M, H)
    cp = cp.double().numpy()
    c_out = torch.full((M, ldc), float('nan'), device='cuda')
    h_f = torch.full((M, ldc), float('nan'), device='cuda')
    hp = torch.zeros(2, M, ldc, dtype=torch.float16, device='cuda')
    epi.lstm, epi.H = 1, H
    epi.c_out, epi.ld_cout = L.ptr(c_out), ldc
    epi.h_f, epi.ld_h = L.ptr(h_f), ldc
    if opt.get('planes'):
        epi.h_hi, epi.h_lo = L.ptr(hp[0]), L.ptr(hp[1])
    L.check(lib.capb200_decode_gemm(L.ptr(xd), L.ptr(wd), M, N, K, L.OP_MODES['tc_f16x3'], epi, None, 0, L.current_stream()),
            'decode_gemm')
    torch.cuda.synchronize()
    sig = lambda v: 1.0 / (1.0 + np.exp(-v))
    zi, zf, zg, zo = (z64[:, q::4] for q in range(4))
    c_ref = sig(zf) * cp + sig(zi) * np.tanh(zg)
    h_ref = sig(zo) * np.tanh(c_ref)
    # Error bar.  Each gate pre-activation is off by at most `tol` (the linear bar above); sigmoid' <= 1/4 and tanh' <= 1, and each
    # fast_sigmoid / fast_tanh adds at most EPS_FAST.  With |sigmoid| <= 1, |tanh| <= 1:
    #   |dc| <= (tol/4 + EPS) |c_prev| + (tol/4 + EPS) + (tol + EPS)
    #   |dh| <= (tol/4 + EPS) + |dc| + EPS
    cmax = float(np.abs(cp).max())
    tol_c = (tol / 4 + EPS_FAST) * cmax + (tol / 4 + EPS_FAST) + (tol + EPS_FAST)
    tol_h = (tol / 4 + EPS_FAST) + tol_c + EPS_FAST
    co, ho = c_out.cpu(), h_f.cpu()
    assert torch.isnan(co[:, H:]).all() and torch.isnan(ho[:, H:]).all()
    err_c = float(np.abs(co[:, :H].double().numpy() - c_ref).max())
    err_h = float(np.abs(ho[:, :H].double().numpy() - h_ref).max())
    assert err_c < tol_c and err_h < tol_h, (shape, opt, err_c, tol_c, err_h, tol_h)
    if opt.get('planes'):
        _check_planes(hp[0, :, :H].cpu(), hp[1, :, :H].cpu(), ho[:, :H])
    else:
        assert not hp.any()
