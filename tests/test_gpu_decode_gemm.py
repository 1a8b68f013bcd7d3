"""GPU: the decode GEMM (tc_f16x3) against fp64 on shapes that reach every tile width (64, 128, 160 columns), ragged and odd m-tile
counts, N that is not a multiple of the tile width and K that is not a multiple of the 64-wide K-block."""
import pytest
import torch

pytestmark = pytest.mark.gpu

# Tile widths noted for an H100 SXM (132 SMs, 66 resident CTA pairs); an odd number of m-tiles leaves the second CTA of the last
# pair without rows of its own.
SHAPES = [
    (1280, 4000, 3000),   # language-LSTM gates of the decode step: BN 160, N a multiple of 160
    (1152, 4000, 1000),   # BN 160 with 9 m-tiles
    (130, 9488, 1000),    # BN 160, ragged second m-tile and ragged last n-tile (9488 is not a multiple of 160)
    (1280, 9488, 1000),   # logit: BN 128, ragged last n-tile
    (1408, 4040, 1000),   # BN 128 with 11 m-tiles
    (1280, 512, 1000),    # h2att: BN 64
    (100, 4040, 1000),    # BN 64, one ragged m-tile
    (256, 4000, 2000),    # BN 64, 2 m-tiles
    (1280, 4000, 72),     # K not a multiple of 64: one full and one partial K-block
]


@pytest.fixture(scope='module')
def L():
    import imagecaptioning.pytorch_b200 as b200
    return b200._lib


def test_tile_widths_cover_every_kernel(L):
    if torch.cuda.get_device_properties(0).multi_processor_count != 132:
        pytest.skip('the widths noted in SHAPES are those of a 132-SM H100 SXM; the choice follows the SM count')
    lib = L.load()
    assert {lib.capb200_gemm_tile_n(M, N) for M, N, _ in SHAPES} == {64, 128, 160}


@pytest.mark.parametrize('shape', SHAPES)
def test_decode_gemm_matches_fp64(L, shape):
    M, N, K = shape
    g = torch.Generator().manual_seed(M * 7 + N + K)
    x = torch.randn(M, K, generator=g)
    w = (torch.rand(N, K, generator=g) * 2 - 1) / K ** 0.5
    b = torch.randn(N, generator=g)
    ref = x.double() @ w.double().t() + b.double()
    xd, wd, bd = x.cuda(), w.cuda(), b.cuda()
    y = torch.empty(M, N, device='cuda')
    L.check(L.load().capb200_linear(L.ptr(xd), K, L.ptr(wd), K, L.ptr(bd), L.ptr(y), N, M, N, K, 0, L.OP_MODES['tc_f16x3'], L.current_stream()),
            'linear')
    torch.cuda.synchronize()
    err = float((y.cpu().double() - ref).abs().max())
    fp32_err = float(((x @ w.t() + b).double() - ref).abs().max())
    # the bar of the operator-level linear test: summation-order noise of fp32 plus one fp32 ulp of the largest output per accumulate
    tol = max(4 * fp32_err, 2e-6) + 3 * (K / 16) * 2.0 ** -24 * float(ref.abs().max())
    assert err < tol, (shape, err, tol)
