"""The multi-head attention operations at any region count (capb200_mha_forward / _self_backward / _cross_backward) against torch float64:
refiner / encoder self-attention (decode form and training form with probability dropout), its backward, and the decoders' attention
backward over the regions.  R runs from 1 to 1024 at head widths 64, 96 and 128 with prefix key masks of 1..R valid regions; dropout masks
are replayed through capb200_dropout_mask.  Where the staged kernel fits, the automatic form must be it bit for bit and the key-tiled form
must agree with it within the bound; the key-tiled form is bitwise reproducible."""
import pytest
import torch

pytestmark = pytest.mark.gpu

HEADS = 8
TOL = 2e-5            # of the largest reference entry (DESIGN.md, 'Region counts')
RS = [1, 7, 36, 75, 76, 105, 106, 196, 577, 1024]
DKS = [64, 96, 128]
LIMIT = 200 * 1024    # bytes of shared memory a staged kernel may use


def _lib():
    import imagecaptioning.pytorch_b200 as b200
    return b200._lib, b200._lib.load()


def _staged_fits(kind, R, dk, rows=0):
    f = {'decode': 2 * R * (dk + 1) + 8 * R + 8 * dk, 'train': 2 * R * (dk + 4) + 8 * R + 8 * dk, 'self_bwd': 4 * R * (dk + 4) + 2 * R * R,
         'cross_bwd': 2 * R * (dk + 1) + 2 * rows * (dk + 1) + 2 * rows * R}[kind]
    return 4 * f <= LIMIT


def _dropout(seed, site, step, shape, p):
    L, lib = _lib()
    n = 1
    for s in shape:
        n *= s
    m = torch.empty(n, device='cuda')
    L.check(lib.capb200_dropout_mask(L.ptr(m), n, seed, site, step, p, L.current_stream()), 'dropout_mask')
    return m.view(*shape)


def _prefix_masks(B, R):
    lens = [1 + (i * (R - 1)) // max(B - 1, 1) for i in range(B)][::-1]       # R valid regions down to 1
    m = torch.zeros(B, R, device='cuda')
    for i, n in enumerate(lens):
        m[i, :n] = 1
    return m


def _err(x, ref):
    """Largest error over the largest reference entry; a reference that is zero (one visible key: no gradient reaches q or k) counts as 1e-3,
    a hundredth of the inputs' scale."""
    return float((x.double() - ref).abs().max()) / max(float(ref.abs().max()), 1e-3)


def _heads(x, B, R, dk):          # [B*R, H] -> [B, heads, R, dk] float64
    return x.double().view(B, R, HEADS, dk).permute(0, 2, 1, 3)


def _unheads(x):                  # [B, heads, R, dk] -> [B*R, H]
    B, h, R, dk = x.shape
    return x.permute(0, 2, 1, 3).reshape(B * R, h * dk)


def _forward(form, train, q, k, v, mask, B, R, dk, seed, site, p):
    L, lib = _lib()
    H = HEADS * dk
    out = torch.full((B * R, H), float('nan'), device='cuda')
    L.check(lib.capb200_mha_forward(form, train, B, R, HEADS, dk, L.ptr(q), L.ptr(k), L.ptr(v), H, L.ptr(mask), R, seed, site, p, L.ptr(out), H,
                                    L.current_stream()), 'mha_forward')
    return out


def _self_backward(form, q, k, v, mask, d_out, B, R, dk, seed, site, p):
    L, lib = _lib()
    H = HEADS * dk
    dq, dk_, dv = (torch.full((B * R, H), float('nan'), device='cuda') for _ in range(3))
    L.check(lib.capb200_mha_self_backward(form, B, R, HEADS, dk, L.ptr(q), L.ptr(k), L.ptr(v), H, L.ptr(mask), R, seed, site, p, L.ptr(d_out), H,
                                          L.ptr(dq), L.ptr(dk_), L.ptr(dv), H, L.current_stream()), 'mha_self_backward')
    return dq, dk_, dv


@pytest.mark.parametrize('dk', DKS)
@pytest.mark.parametrize('R', RS)
def test_self_attention_forward_and_backward(R, dk):
    """Decode-form and training-form forward and the backward of the refiner / encoder self-attention, p in {0, 0.1}, prefix masks."""
    L, lib = _lib()
    B = 4 if R < 577 else 2
    H = HEADS * dk
    g = torch.Generator(device='cuda').manual_seed(R * 1000 + dk)
    q, k, v, d_out = (torch.randn(B * R, H, device='cuda', generator=g) for _ in range(4))
    mask = _prefix_masks(B, R)
    scale = dk ** -0.5
    qh, kh, vh = (_heads(x, B, R, dk).requires_grad_(True) for x in (q, k, v))
    s = (qh @ kh.transpose(-1, -2)) * scale
    s = s.masked_fill(mask.view(B, 1, 1, R) == 0, float('-inf'))
    P = torch.softmax(s, -1)
    for p in (0.0, 0.1):
        seed, site = 1234 + int(p * 10), 11
        for train in ((0, 1) if p == 0 else (1,)):
            kind = 'train' if train else 'decode'
            Z = _dropout(seed, site, 0, (B, HEADS, R, R), p).double() if train else 1.0
            ref = _unheads((P * Z) @ vh).detach()
            o2 = _forward(2, train, q, k, v, mask, B, R, dk, seed, site, p)
            assert _err(o2, ref) <= TOL, (kind, p, _err(o2, ref))
            assert torch.equal(o2, _forward(2, train, q, k, v, mask, B, R, dk, seed, site, p))
            o0 = _forward(0, train, q, k, v, mask, B, R, dk, seed, site, p)
            if _staged_fits(kind, R, dk):
                o1 = _forward(1, train, q, k, v, mask, B, R, dk, seed, site, p)
                assert torch.equal(o0, o1)
                assert _err(o1, ref) <= TOL
            else:
                assert torch.equal(o0, o2)
                with pytest.raises(RuntimeError):
                    _forward(1, train, q, k, v, mask, B, R, dk, seed, site, p)
        # backward of the training form
        Z = _dropout(seed, site, 0, (B, HEADS, R, R), p).double()
        out = (P * Z) @ vh
        gq, gk, gv = torch.autograd.grad(out, (qh, kh, vh), _heads(d_out, B, R, dk), retain_graph=True)
        refs = [_unheads(x) for x in (gq, gk, gv)]
        b2 = _self_backward(2, q, k, v, mask, d_out, B, R, dk, seed, site, p)
        for x, ref in zip(b2, refs):
            assert _err(x, ref) <= TOL, (p, _err(x, ref))
        assert all(torch.equal(a, b) for a, b in zip(b2, _self_backward(2, q, k, v, mask, d_out, B, R, dk, seed, site, p)))
        b0 = _self_backward(0, q, k, v, mask, d_out, B, R, dk, seed, site, p)
        if _staged_fits('self_bwd', R, dk):
            b1 = _self_backward(1, q, k, v, mask, d_out, B, R, dk, seed, site, p)
            assert all(torch.equal(a, b) for a, b in zip(b0, b1))
            for x, ref in zip(b1, refs):
                assert _err(x, ref) <= TOL
        else:
            assert all(torch.equal(a, b) for a, b in zip(b0, b2))


def _cross_backward(form, q, kk, vv, probs, d_out, B, rpi, T, R, dk, seed, site, step, p, dk0, dv0):
    L, lib = _lib()
    H = HEADS * dk
    dq = torch.full_like(q, float('nan'))
    dkk, dvv = dk0.clone(), dv0.clone()
    L.check(lib.capb200_mha_cross_backward(form, B, rpi, T, HEADS, dk, R, L.ptr(q), H, L.ptr(kk), L.ptr(vv), H, seed, site, step, p, L.ptr(probs),
                                           L.ptr(d_out), H, L.ptr(dq), H, L.ptr(dkk), L.ptr(dvv), H, L.current_stream()), 'mha_cross_backward')
    return dq, dkk, dvv


@pytest.mark.parametrize('dk', DKS)
@pytest.mark.parametrize('R', RS)
@pytest.mark.parametrize('rpi,T', [(5, 1), (16, 1), (5, 17), (16, 21)])
def test_cross_attention_backward(R, dk, rpi, T):
    """The decoders' attention over the regions: rows TIME-major (T blocks of B * rpi rows), probabilities from the tape, dK / dV added."""
    B = 3
    H = HEADS * dk
    rows = T * B * rpi
    g = torch.Generator(device='cuda').manual_seed(R * 7 + dk + rpi * 1000 + T)
    q, d_out = (torch.randn(rows, H, device='cuda', generator=g) for _ in range(2))
    kk, vv, dk0, dv0 = (torch.randn(B * R, H, device='cuda', generator=g) for _ in range(4))
    mask = _prefix_masks(B, R)
    scale = dk ** -0.5
    # rows [T, B, rpi] x heads against the image's keys
    qh = q.double().view(T, B, rpi, HEADS, dk).permute(1, 3, 0, 2, 4).reshape(B, HEADS, T * rpi, dk).requires_grad_(True)
    kh, vh = (x.double().view(B, R, HEADS, dk).permute(0, 2, 1, 3).requires_grad_(True) for x in (kk, vv))
    s = ((qh @ kh.transpose(-1, -2)) * scale).masked_fill(mask.view(B, 1, 1, R) == 0, float('-inf'))
    P = torch.softmax(s, -1)
    # probs as cross_attn_train_kernel saves them: [(row * heads + head), R]
    probs = P.detach().float().view(B, HEADS, T, rpi, R).permute(2, 0, 3, 1, 4).reshape(rows * HEADS, R).contiguous()
    dOh = d_out.double().view(T, B, rpi, HEADS, dk).permute(1, 3, 0, 2, 4).reshape(B, HEADS, T * rpi, dk)
    for p in (0.0, 0.1):
        seed, site, step = 99 + int(p * 10), 5, 3
        # dropout element (b * rpi + j) * heads + h) * R + r at step `step` + t
        Z = torch.stack([_dropout(seed, site, step + t, (B, rpi, HEADS, R), p) for t in range(T)])         # [T, B, rpi, heads, R]
        Zh = Z.double().permute(1, 3, 0, 2, 4).reshape(B, HEADS, T * rpi, R)
        gq, gk, gv = torch.autograd.grad((P * Zh) @ vh, (qh, kh, vh), dOh, retain_graph=True)
        ref_q = gq.view(B, HEADS, T, rpi, dk).permute(2, 0, 3, 1, 4).reshape(rows, H)
        ref_k = dk0.double() + gk.permute(0, 2, 1, 3).reshape(B * R, H)
        ref_v = dv0.double() + gv.permute(0, 2, 1, 3).reshape(B * R, H)
        r2 = _cross_backward(2, q, kk, vv, probs, d_out, B, rpi, T, R, dk, seed, site, step, p, dk0, dv0)
        assert _err(r2[0], ref_q) <= TOL, (p, _err(r2[0], ref_q))
        # dK / dV relative to the gradient added, not to the buffers they are added into
        assert float((r2[1].double() - ref_k).abs().max()) <= TOL * float(gk.abs().max()) + 1e-6
        assert float((r2[2].double() - ref_v).abs().max()) <= TOL * float(gv.abs().max()) + 1e-6
        again = _cross_backward(2, q, kk, vv, probs, d_out, B, rpi, T, R, dk, seed, site, step, p, dk0, dv0)
        assert all(torch.equal(a, b) for a, b in zip(r2, again))
        r0 = _cross_backward(0, q, kk, vv, probs, d_out, B, rpi, T, R, dk, seed, site, step, p, dk0, dv0)
        if _staged_fits('cross_bwd', R, dk, rpi * T):
            r1 = _cross_backward(1, q, kk, vv, probs, d_out, B, rpi, T, R, dk, seed, site, step, p, dk0, dv0)
            assert all(torch.equal(a, b) for a, b in zip(r0, r1))
            assert _err(r1[0], ref_q) <= TOL
        else:
            assert all(torch.equal(a, b) for a, b in zip(r0, r2))


def test_dropout_index_bound():
    """The 32-bit dropout index: a training-form launch with B * heads * R^2 >= 2^32 elements is refused with a message, not wrapped."""
    L, lib = _lib()
    B, R, dk = 128, 2048, 4
    x = torch.zeros(B * R, HEADS * dk, device='cuda')
    rc = lib.capb200_mha_forward(2, 1, B, R, HEADS, dk, L.ptr(x), L.ptr(x), L.ptr(x), HEADS * dk, None, 0, 1, 11, 0.1, L.ptr(x), HEADS * dk,
                                 L.current_stream())
    assert rc != 0
    assert '2^32' in lib.capb200_last_error().decode()
