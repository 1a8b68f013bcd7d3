"""The decode GEMM's cooperative schedule (gemm_tc256_kernel: 256 x BN tiles, both consumer warpgroups reading one weight tile).

GPU: with CAPB200_GEMM_BM=256 forcing it, every epilogue kind at BN 128 and 160 against float64, and bitwise equal to the 128-row
ping-pong schedule (CAPB200_GEMM_BM=128) on the same inputs: both run the same wgmmas in the same order per output element.  M covers
one m-tile, a second m-tile of one row (its upper 128-row half wholly past the rows), ragged and many m-tiles; N is ragged against the
tile width and K against the 64-wide K-block.  A whole UpDown beam search, whose gate GEMMs walk two and three K-segments and whose
t = 0 launches run fewer rows than their plans (M override), gives the same ids and log-probabilities under both schedules.
CPU: the machine code of every production gemm_tc256_kernel stays under the ceiling test_decode_gemm_code_size.py sets for the 128-row
kernels."""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from test_decode_gemm_code_size import CEILING_KB, LIB, _cuobjdump

EPS_FAST = 1e-6   # fast_sigmoid / fast_tanh absolute error (common.cuh), as in test_gpu_decode_gemm_epilogue.py
KERNEL256 = re.compile(r'gemm_tc256_kernelILi(\d+)ELi(\d+)ELi(\d+)ELb([01])E')
CASES = [
    ('store', dict(bias=True, relu=True, residual=True)),
    ('planes', dict(bias=True, row_bias=True, odd_pitch=True)),
    ('lstm', dict(row_bias=True, gather=True, src='permuted', planes=True)),      # attention LSTM of the decode step
    ('lstm', dict(bias=True, residual=True, relu=True, src='identity')),
]
ROWS = [256, 257, 300, 1280, 9216]


class _Schedule:
    """CAPB200_GEMM_BM for the launches inside the block (the library reads it at every launch)."""

    def __init__(self, bm):
        self.bm = bm

    def __enter__(self):
        self.old = os.environ.get('CAPB200_GEMM_BM')
        os.environ['CAPB200_GEMM_BM'] = str(self.bm)

    def __exit__(self, *exc):
        if self.old is None:
            os.environ.pop('CAPB200_GEMM_BM', None)
        else:
            os.environ['CAPB200_GEMM_BM'] = self.old


@pytest.fixture(scope='module')
def L():
    import imagecaptioning.pytorch_b200 as b200
    return b200._lib


def _ragged_n(lib, M, bn):
    # the first N (a multiple of 4 for the LSTM kind, not of bn) for which the plan picks width bn on this device
    for N in range(1000, 20000, 4):
        if N % bn and lib.capb200_gemm_tile_n(M, N) == bn:
            return N
    pytest.skip('no N up to 20000 takes width %d at M = %d on this device' % (bn, M))


def _launch(L, lib, xd, wd, M, N, K, epi, bm):
    with _Schedule(bm):
        assert lib.capb200_gemm_tile_m(M, N) == bm
        L.check(lib.capb200_decode_gemm(L.ptr(xd), L.ptr(wd), M, N, K, L.OP_MODES['tc_f16x3'], epi, None, 0, L.current_stream()),
                'decode_gemm')
    torch.cuda.synchronize()


@pytest.mark.gpu
@pytest.mark.parametrize('kind,opt', CASES, ids=['%s%d' % (k, i) for i, (k, _) in enumerate(CASES)])
@pytest.mark.parametrize('bn', [128, 160])
@pytest.mark.parametrize('M', ROWS)
def test_256_rows_match_fp64_and_128_rows(L, M, bn, kind, opt):
    lib = L.load()
    N = _ragged_n(lib, M, bn)
    K = 136 + 64 * (M % 3)                     # 3 to 5 K-blocks, the last one partial
    g = torch.Generator().manual_seed(M + 3 * N + K + len(opt))
    x = torch.randn(M, K, generator=g)
    w = (torch.rand(N, K, generator=g) * 2 - 1) / K ** 0.5
    xd, wd = x.cuda(), w.cuda()
    epi = L.GemmEpilogue()
    keep = []

    def dev(t):
        t = t.cuda()
        keep.append(t)
        return L.ptr(t)

    z64 = x.double() @ w.double().t()
    z32 = x @ w.t()
    if opt.get('bias'):
        b = torch.randn(N, generator=g)
        epi.bias = dev(b)
        z64 += b.double(); z32 += b
    if opt.get('row_bias'):
        rb = torch.randn(-(-M // 5), N + 3, generator=g)
        epi.row_bias, epi.ld_row_bias, epi.rows_per_group = dev(rb), N + 3, 5
        rows = torch.arange(M) // 5
        z64 += rb[rows, :N].double(); z32 += rb[rows, :N]
    if opt.get('gather'):
        tab = torch.randn(7, N + 5, generator=g)
        idx = torch.randint(0, 7, (M,), generator=g, dtype=torch.int32)
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
    # the bar of test_gpu_decode_gemm.py: summation-order noise of fp32 plus one fp32 ulp of the largest output per accumulate
    tol = max(4 * float(np.abs(z32.double().numpy() - z64).max()), 2e-6) + 3 * (K / 16) * 2.0 ** -24 * float(np.abs(z64).max())
    pad = 1 if opt.get('odd_pitch') else 0

    if kind in ('store', 'planes'):
        ld = N + pad
        outs = {}
        for bm in (256, 128):
            y = torch.full((M, ld), float('nan'), device='cuda')
            planes = torch.zeros(2, M, ld, dtype=torch.float16, device='cuda')
            epi.C, epi.ldc = L.ptr(y), ld
            if kind == 'planes':
                epi.C_hi, epi.C_lo, epi.ldcs = L.ptr(planes[0]), L.ptr(planes[1]), ld
            _launch(L, lib, xd, wd, M, N, K, epi, bm)
            outs[bm] = (y.cpu(), planes.cpu())
        y, planes = outs[256]
        assert torch.isnan(y[:, N:]).all()
        err = float(np.abs(y[:, :N].double().numpy() - z64).max())
        assert err < tol, (M, N, K, kind, err, tol)
        if kind == 'planes':
            assert torch.equal(planes[0, :, :N], y[:, :N].half()) and torch.equal(planes[1, :, :N], (y[:, :N] - planes[0, :, :N].float()).half())
        assert torch.equal(outs[128][0].nan_to_num(7.0), y.nan_to_num(7.0)) and torch.equal(outs[128][1], planes)
        return

    H = N // 4
    c_prev = torch.randn(M, H, generator=g)
    if opt.get('src') == 'permuted':
        srow = torch.randperm(M, generator=g).int()
        srow[::7] = -1                                                   # fresh rows start from the zero state
        epi.src_row = dev(srow)
        cp = torch.where((srow >= 0)[:, None], c_prev[srow.long().clamp_min(0)], torch.zeros(()))
    else:
        cp = c_prev
    cp = cp.double().numpy()
    epi.c_prev, epi.ld_cprev = dev(c_prev), H
    epi.lstm, epi.H = 1, H
    outs = {}
    for bm in (256, 128):
        c_out = torch.full((M, H), float('nan'), device='cuda')
        h_f = torch.full((M, H), float('nan'), device='cuda')
        hp = torch.zeros(2, M, H, dtype=torch.float16, device='cuda')
        epi.c_out, epi.ld_cout = L.ptr(c_out), H
        epi.h_f, epi.ld_h = L.ptr(h_f), H
        if opt.get('planes'):
            epi.h_hi, epi.h_lo = L.ptr(hp[0]), L.ptr(hp[1])
        _launch(L, lib, xd, wd, M, N, K, epi, bm)
        outs[bm] = (c_out.cpu(), h_f.cpu(), hp.cpu())
    sig = lambda v: 1.0 / (1.0 + np.exp(-v))
    zi, zf, zg, zo = (z64[:, q::4] for q in range(4))
    c_ref = sig(zf) * cp + sig(zi) * np.tanh(zg)
    h_ref = sig(zo) * np.tanh(c_ref)
    cmax = float(np.abs(cp).max())
    tol_c = (tol / 4 + EPS_FAST) * cmax + (tol / 4 + EPS_FAST) + (tol + EPS_FAST)
    tol_h = (tol / 4 + EPS_FAST) + tol_c + EPS_FAST
    c_out, h_f, hp = outs[256]
    err_c = float(np.abs(c_out.double().numpy() - c_ref).max())
    err_h = float(np.abs(h_f.double().numpy() - h_ref).max())
    assert err_c < tol_c and err_h < tol_h, (M, N, K, opt, err_c, tol_c, err_h, tol_h)
    if opt.get('planes'):
        assert torch.equal(hp[0], h_f.half()) and torch.equal(hp[1], (h_f - hp[0].float()).half())
    for a, b in zip(outs[128], outs[256]):
        assert torch.equal(a, b)


@pytest.mark.gpu
def test_updown_beam_search_same_under_both_schedules():
    # 64 images x beam 5 = 320 rows: the gate and logit plans take widths 128 / 160, so CAPB200_GEMM_BM=256 reaches every fused epilogue
    from imagecaptioning.pytorch_b200 import synthetic as syn
    cfg = dict(V=9487, E=1000, H=1000, A=512, F_fc=2048, F_att=2048, T=12)
    fc, att = syn.make_inputs(64, 36, 2048, 2048, seed=5)
    fc, att = fc.cuda(), att.cuda()
    outs = {}
    for bm in (256, 128):
        with _Schedule(bm):
            model = syn.build_model('updown', seed=5, logit_scale=12.0, mode='tc_f16x3', **cfg)
            with torch.no_grad():
                seq, lp = model(fc, att, None, opt={'beam_size': 5, 'sample_n': 1}, mode='sample')
            torch.cuda.synchronize()
        outs[bm] = (seq.cpu(), lp.cpu())
        del model
    assert torch.equal(outs[128][0], outs[256][0])
    assert torch.equal(outs[128][1], outs[256][1])


def test_256_row_kernels_fit_the_ceiling():
    tool = _cuobjdump()
    if tool is None or not os.path.exists(LIB):
        pytest.skip('needs cuobjdump and the built library')
    sass = subprocess.run([tool, '-sass', LIB], capture_output=True, text=True, check=True).stdout
    sizes = {}
    for chunk in re.split(r'\n\s*Function : ', sass)[1:]:
        m = KERNEL256.search(chunk.split('\n', 1)[0])
        if m is None or m.group(4) == '1':           # TRACE = true: the diagnostic build of tools/gemm_trace.py
            continue
        sizes['BN %s, %s-pass, kind %s' % m.groups()[:3]] = len(re.findall(r'/\*[0-9a-f]{4,}\*/\s+[^;\n]*;', chunk)) * 16
    assert len(sizes) == 3 * 2 * 2, sorted(sizes)     # kind x BN (128, 160) x passes
    over = {k: v for k, v in sizes.items() if v > CEILING_KB * 1024}
    assert not over, over
