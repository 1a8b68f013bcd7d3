"""The vocabulary step above one CTA's shared memory: V + 1 = 51 201 .. 409 600 entries, where every row is spread over a
thread-block cluster (vocab_step_cluster_kernel in csrc/vocab.cu), against float64, through the operator-level entry points
capb200_vocab_select (greedy, multinomial, top-k, nucleus), capb200_log_softmax_topk (the k-round top-k list) and
capb200_vocab_stats_topk (beam search's statistics kernel, which streams the row and has no length limit).

The draws are predicted exactly: philox_first below restates the kernel's generator in numpy (checked on the CPU against the
Random123 known-answer vectors), so each multinomial / top-k / nucleus draw is the float64 arg-max of logp / T - log(-log u) over the
kept words, wherever the best key is clear of the second by more than 1e-5.

Largest errors against float64 observed on one H100 (80 GB HBM3, 700 W) are printed at teardown (pytest -s).
"""
import numpy as np
import pytest
import torch

SENTINEL = 0x7fffffff
NEG_INF = float('-inf')
HAS_GPU = torch.cuda.is_available()
TOL = 5e-6                      # log-sum-exp and candidate log-probs against float64
TOL_ROW = 1e-5                  # the sampling kernel's stored row and picked log-prob
ULP = 2.0 ** -23
SLICE = 51200                   # entries one CTA of the cluster caches
MAX_ROW = 8 * SLICE
GREEDY, MULTINOMIAL, TOPK, NUCLEUS = 1, 2, 4, 5

OBSERVED = {}


def gpu(fn):
    return pytest.mark.gpu(pytest.mark.skipif(not HAS_GPU, reason='needs a CUDA device')(fn))


def _note(name, v):
    OBSERVED[name] = max(OBSERVED.get(name, 0.0), float(v))


@pytest.fixture(scope='module')
def L():
    import imagecaptioning.pytorch_b200 as b200
    L = b200._lib
    # a graph replay of a training step elsewhere in the process may have left a seed salt behind; this entry point clears it
    m = torch.empty(4, device='cuda')
    L.check(L.load().capb200_dropout_mask(L.ptr(m), 4, 1, 0, 0, 0.5, L.current_stream()), 'dropout_mask')
    torch.cuda.synchronize()
    yield L
    if OBSERVED:
        print('\n[large vocab step] largest errors against float64: ' + ', '.join('%s %.3g' % kv for kv in sorted(OBSERVED.items())))


def slices(V1):
    """[lo, hi) of each CTA of the row's cluster."""
    C = -(-V1 // SLICE)
    S = -(-V1 // C)
    return [(c * S, min(V1, (c + 1) * S)) for c in range(C)]


# ---------------------------------------------------------------------------------------------------------------------------------
# Philox4x32-10, restated
# ---------------------------------------------------------------------------------------------------------------------------------
M0, M1, W0, W1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57), np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
MASK = np.uint64(0xffffffff)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """All four output words of Philox4x32-10 (Salmon et al. 2011), elementwise over broadcast uint32 arrays."""
    c = [np.asarray(x, dtype=np.uint32) for x in (c0, c1, c2, c3)]
    k0, k1 = np.uint32(k0), np.uint32(k1)
    with np.errstate(over='ignore'):
        for _ in range(10):
            p0 = M0 * c[0].astype(np.uint64)
            p1 = M1 * c[2].astype(np.uint64)
            hi0, lo0 = (p0 >> np.uint64(32)).astype(np.uint32), (p0 & MASK).astype(np.uint32)
            hi1, lo1 = (p1 >> np.uint64(32)).astype(np.uint32), (p1 & MASK).astype(np.uint32)
            c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
            k0 = np.uint32(k0 + W0)
            k1 = np.uint32(k1 + W1)
    return c


def gumbel_u(V1, rows, step, seed):
    """The kernel's uniform for every (row, word): philox_first(word, row, step lo, step hi, seed lo, seed hi), 23 bits, in (0, 1)."""
    w = np.arange(V1, dtype=np.uint32)[None, :]
    r = np.asarray(rows, dtype=np.uint32)[:, None]
    bits = philox4x32_10(w, r, np.uint32(step & 0xffffffff), np.uint32(step >> 32), seed & 0xffffffff, seed >> 32)[0]
    return ((bits >> np.uint32(9)).astype(np.float64) + 0.5) * (1.0 / 8388608.0)


def test_philox_restatement_known_answers():
    """Random123's known-answer vectors for philox4x32-10."""
    kat = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
           ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
           ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, out in kat:
        got = philox4x32_10(*ctr, *key)
        assert [int(x) for x in got] == list(out)


def test_slices_cover_the_row():
    for V1 in (51201, 60001, 65536, 100001, 131072, 262147, 409600):
        s = slices(V1)
        assert s[0][0] == 0 and s[-1][1] == V1 and len(s) <= 8
        assert all(a[1] == b[0] for a, b in zip(s, s[1:])) and all(hi - lo <= SLICE and hi > lo for lo, hi in s)


# ---------------------------------------------------------------------------------------------------------------------------------
# float64 references (computed on the device: the rows are large)
# ---------------------------------------------------------------------------------------------------------------------------------
def ref_logp(x):
    xd = x.double()
    return xd - torch.logsumexp(xd, -1, keepdim=True)


def ref_order(x, k):
    """value descending, lowest column first on ties"""
    return torch.sort(x, dim=-1, descending=True, stable=True).indices[..., :k]


def place(x, layout):
    """rows of x on the device; every float around them holds +1e30 (a read outside a row finds a wrong maximum)."""
    rows, V1 = x.shape
    if layout == 'dense':
        buf = x.to('cuda', copy=True).contiguous()
        return buf, buf, V1
    if layout in ('pitch4', 'pitch1'):
        ld = V1 + (4 if layout == 'pitch4' else 1)
        buf = torch.full((rows, ld), 1e30, device='cuda')
        buf[:, :V1] = x
        return buf, buf[:, :V1], ld
    buf = torch.full((rows * V1 + 4,), 1e30, device='cuda')
    view = buf[1:1 + rows * V1].view(rows, V1)
    view.copy_(x)
    return buf, view, V1


def run_select(L, x, select, top=0.0, temperature=1.0, seed=1234, step=0, unfinished=None, first_step=1, layout='dense'):
    """Returns tokens, picked log-probs, the rewritten rows and the whole buffer (device tensors)."""
    rows, V1 = x.shape
    buf, view, ld = place(x, layout)
    tokens = torch.full((rows,), -7, dtype=torch.int32, device='cuda')
    picked = torch.full((rows,), 7.0, device='cuda')
    L.check(L.load().capb200_vocab_select(L.ptr(view), ld, rows, V1, select, top, temperature, seed, step, L.ptr(unfinished), first_step,
                                          L.ptr(tokens), L.ptr(picked), L.current_stream()), 'vocab_select')
    torch.cuda.synchronize()
    return tokens, picked, view, buf


def row_error(row, lp):
    """|row - float64| less the rounding of the fp32 result itself (rows reaching -1e3 and below carry ulps of 1e-4)"""
    fin = torch.isfinite(lp)
    assert torch.equal(torch.isfinite(row.double()), fin)
    return float(((row.double() - lp).abs() - 4 * ULP * lp.abs())[fin].max())


def plant(V1, rows, where, seed, k=16):
    """Random rows whose k largest values sit in `where`: 'one' = all inside the second CTA's slice, 'boundary' = alternating on both
    sides of the first slice boundary, 'last' = the last k columns."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, V1, generator=g) * 3
    lo, hi = slices(V1)[1] if len(slices(V1)) > 1 else slices(V1)[0]
    b = slices(V1)[0][1]
    for r in range(rows):
        if where == 'one':
            cols = (lo + torch.randperm(hi - lo, generator=g)[:k]).tolist()
        elif where == 'boundary':
            cols = [b - 1 - i // 2 if i % 2 == 0 else b + i // 2 for i in range(k)]
        else:
            cols = list(range(V1 - k, V1))
        vals = 20.0 + 0.25 * torch.randperm(k, generator=g).float()
        x[r, torch.tensor(cols)] = vals
    return x


SIZES = [51201, 60001, 65536, 131072, 262147, 409600]


def rows_for(V1):
    return (1, 17, 1280) if V1 <= 131072 else (1, 17)


# ---------------------------------------------------------------------------------------------------------------------------------
# A. greedy: log-softmax rows, the stable arg-max, layouts and value ranges
# ---------------------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('V1', SIZES)
def test_greedy_rows_and_argmax(L, V1):
    for rows in rows_for(V1):
        g = torch.Generator(device='cuda').manual_seed(V1 + rows)
        x = torch.randn(rows, V1, generator=g, device='cuda') * 4
        x[0, [7, V1 // 2, V1 - 1]] = 30.0                           # tied maxima in different CTAs: the lowest column wins
        tokens, picked, row, _ = run_select(L, x, GREEDY)
        lp = ref_logp(x)
        assert torch.equal(tokens.long(), ref_order(x, 1)[:, 0]), (V1, rows)
        assert int(tokens[0]) == 7
        e_pick = float((picked.double() - lp.gather(1, tokens.long()[:, None])[:, 0]).abs().max())
        e_row = row_error(row, lp)
        _note('picked_lp', e_pick)
        _note('row', e_row)
        assert e_pick < TOL_ROW and e_row < TOL_ROW, (V1, rows, e_pick, e_row)


@gpu
@pytest.mark.parametrize('layout', ['pitch4', 'pitch1', 'offset1'])
@pytest.mark.parametrize('V1', [51201, 65536, 409600])
def test_greedy_pitched_and_misaligned(L, V1, layout):
    g = torch.Generator(device='cuda').manual_seed(V1 + len(layout))
    x = torch.randn(17, V1, generator=g, device='cuda') * 4
    x[2] = plant(V1, 1, 'boundary', seed=V1 + 1)[0].cuda()
    x[3] = plant(V1, 1, 'last', seed=V1 + 2)[0].cuda()
    tokens, picked, row, buf = run_select(L, x, GREEDY, layout=layout)
    lp = ref_logp(x)
    assert torch.equal(tokens.long(), ref_order(x, 1)[:, 0])
    assert row_error(row, lp) < TOL_ROW
    if layout in ('pitch4', 'pitch1'):
        assert bool((buf[:, V1:] == 1e30).all())
    else:
        assert bool(buf[0] == 1e30) and bool((buf[1 + 17 * V1:] == 1e30).all())


@gpu
@pytest.mark.parametrize('V1', [51201, 131072, 409600])
def test_greedy_value_ranges(L, V1):
    g = torch.Generator(device='cuda').manual_seed(V1)
    base = torch.randn(4, V1, generator=g, device='cuda')
    rows = [base[0] * 1000, base[1] * 4 + 3e4, base[1] * 4 - 3e4, torch.zeros(V1, device='cuda')]
    r = base[2].clone() * 4
    r[torch.randperm(V1, generator=g, device='cuda')[:V1 // 3]] = NEG_INF       # scattered -inf columns
    rows.append(r)
    r = base[3].clone() * 4                                                      # a whole slice at -inf except one column
    lo, hi = slices(V1)[-1]
    r[lo:hi] = NEG_INF
    r[hi - 1] = 2.0
    rows.append(r)
    x = torch.stack(rows)
    tokens, picked, row, _ = run_select(L, x, GREEDY)
    lp = ref_logp(x)
    assert torch.equal(tokens.long(), ref_order(x, 1)[:, 0])
    assert int(tokens[3]) == 0                                                   # an all-equal row picks column 0
    assert row_error(row, lp) < TOL_ROW
    e = (picked.double() - lp.gather(1, tokens.long()[:, None])[:, 0]).abs() - 4 * ULP * lp.gather(1, tokens.long()[:, None])[:, 0].abs()
    assert float(e.max()) < TOL_ROW


# ---------------------------------------------------------------------------------------------------------------------------------
# B. the k-round top-k list of the cluster kernel, and beam search's statistics kernel at the same lengths
# ---------------------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('k', [2, 5, 16])
@pytest.mark.parametrize('V1', SIZES)
def test_topk_list_is_the_stable_sort(L, V1, k):
    """capb200_log_softmax_topk ranks on the rounded log-probs it writes: its list must be the stable sort of that row, bit for bit
    (value descending, lowest column first), and the row must match float64.  Rows put the k best inside one CTA's slice, across a
    slice boundary, on the last columns, and tie them."""
    g = torch.Generator(device='cuda').manual_seed(V1 * 3 + k)
    parts = [torch.randn(5, V1, generator=g, device='cuda') * 4]
    for where in ('one', 'boundary', 'last'):
        parts.append(plant(V1, 2, where, seed=V1 + k + len(where), k=k).cuda())
    tie = torch.randn(3, V1, generator=g, device='cuda')
    tie[0, torch.randperm(V1, generator=g, device='cuda')[:2 * k]] = 9.0        # the top value 2k times, spread over the slices
    tie[1] = 0.0                                                                 # all equal: columns 0 .. k-1
    tie[2, [slices(V1)[0][1] - 1, slices(V1)[0][1], V1 - 1, 3]] = 9.0
    parts.append(tie)
    x = torch.cat(parts)
    rows = x.shape[0]
    xd = x.clone()
    tv = torch.empty(rows, k, device='cuda')
    ti = torch.empty(rows, k, dtype=torch.int32, device='cuda')
    L.check(L.load().capb200_log_softmax_topk(L.ptr(xd), V1, rows, V1, 0, k, L.ptr(tv), L.ptr(ti), L.current_stream()), 'log_softmax_topk')
    torch.cuda.synchronize()
    assert torch.equal(ti.long(), ref_order(xd, k)), V1
    assert torch.equal(tv, xd.gather(1, ti.long()))
    assert row_error(xd, ref_logp(x)) < TOL_ROW
    assert ti[-2].tolist() == list(range(k))
    # twice = 1: the values move by the second normalisation, the order does not
    xd2 = x.clone()
    tv2 = torch.empty(rows, k, device='cuda')
    ti2 = torch.empty(rows, k, dtype=torch.int32, device='cuda')
    L.check(L.load().capb200_log_softmax_topk(L.ptr(xd2), V1, rows, V1, 1, k, L.ptr(tv2), L.ptr(ti2), L.current_stream()), 'log_softmax_topk')
    torch.cuda.synchronize()
    assert torch.equal(ti2, ti)
    lp2 = ref_logp(ref_logp(x))
    assert float((tv2.double() - lp2.gather(1, ti.long())).abs().max()) < TOL


@gpu
@pytest.mark.parametrize('V1', SIZES)
def test_stats_topk_at_large_vocabulary(L, V1):
    for rows in rows_for(V1):
        g = torch.Generator(device='cuda').manual_seed(V1 + 7 * rows)
        x = torch.randn(rows, V1, generator=g, device='cuda') * 4
        k = 16
        stats = torch.empty(rows, 2, device='cuda')
        top_val = torch.empty(rows, k, device='cuda')
        top_idx = torch.empty(rows, k, dtype=torch.int32, device='cuda')
        L.check(L.load().capb200_vocab_stats_topk(L.ptr(x), V1, rows, V1, 1, k, L.ptr(stats), L.ptr(top_val), L.ptr(top_idx),
                                                  L.current_stream()), 'vocab_stats_topk')
        torch.cuda.synchronize()
        xd = x.double()
        mx = xd.max(1).values
        lse = (xd - mx[:, None]).exp().sum(1).log()
        assert torch.equal(stats[:, 0].double(), mx)
        e = float((stats[:, 1].double() - lse).abs().max())
        _note('stats lse', e)
        assert e <= TOL
        assert torch.equal(top_idx.long(), ref_order(x, k))


# ---------------------------------------------------------------------------------------------------------------------------------
# C. samplers: every draw predicted
# ---------------------------------------------------------------------------------------------------------------------------------
def kept(lp, select, top, temperature):
    """Kept words of sample_next_word (CaptionModel.py:375-406) per row, float64; ties at the threshold are all kept."""
    if select == MULTINOMIAL:
        return torch.ones_like(lp, dtype=torch.bool)
    srt, order = torch.sort(lp, dim=1, descending=True, stable=True)
    if select == TOPK:
        k = int(top)
        return lp >= srt[:, k - 1:k] if k < lp.shape[1] else torch.ones_like(lp, dtype=torch.bool)
    q = torch.softmax(srt / temperature, 1)
    cum = torch.cat([torch.zeros_like(q[:, :1]), q.cumsum(1)[:, :-1]], 1)     # mass of the words before each sorted word
    # a word's fate is that of the first word of its tie group: the mass strictly above it
    first = torch.searchsorted(-srt.contiguous(), -srt.contiguous(), right=False)
    keep_sorted = cum.gather(1, first) < top
    keep = torch.zeros_like(keep_sorted)
    keep.scatter_(1, order, keep_sorted)
    return keep, cum.gather(1, first), order


def zipf_rows(V1, exponents, seed):
    g = torch.Generator().manual_seed(seed)
    rows = []
    for s in exponents:
        row = torch.empty(V1)
        row[torch.randperm(V1, generator=g)] = -s * torch.log(torch.arange(1, V1 + 1, dtype=torch.float64)).float()
        rows.append(row + 3.0)
    return torch.stack(rows)


@gpu
@pytest.mark.parametrize('select,top', [(MULTINOMIAL, 0.0), (TOPK, 1.0), (TOPK, 5.0), (TOPK, 50.0), (NUCLEUS, 0.3), (NUCLEUS, 0.9)])
@pytest.mark.parametrize('V1', [51201, 100001, 409600])
def test_draws_match_the_predicted_word(L, V1, select, top):
    """Each draw is the float64 arg-max of logp / T - log(-log u) over the kept words, u from the restated Philox stream; checked on
    every draw whose best key is clear of the second by more than 1e-5 (at least 95% of them)."""
    temperature = 0.7 if select == NUCLEUS else 1.3
    base = zipf_rows(V1, (1.0, 2.4, 3.4), seed=V1)
    if select == MULTINOMIAL:                                     # flat rows too, where nothing has to be cut exactly
        base = torch.cat([base, torch.randn(3, V1, generator=torch.Generator().manual_seed(V1)) * 3])
    rows = 12
    x = base[torch.arange(rows) % base.shape[0]].cuda()
    lp = ref_logp(x)
    if select == NUCLEUS:
        keep, mass, _ = kept(lp, select, top, temperature)
        assert float((mass - top).abs().min()) > 5e-6            # no word on the threshold: fp32 mass sums cannot change the set
    else:
        keep = kept(lp, select, top, temperature)
        if select == TOPK:                                        # the k-th word is clear of the next one
            srt = torch.sort(lp, 1, descending=True).values
            assert float((srt[:, int(top) - 1] - srt[:, int(top)]).min()) > 1e-4
    seed = 0x1234567890ab ^ int(V1)
    checked = total = 0
    for step in (0, 1, 2 ** 32 + 5):
        tokens, picked, _, _ = run_select(L, x, select, top, temperature, seed=seed, step=step)
        u = torch.from_numpy(gumbel_u(V1, np.arange(rows), step, seed)).cuda()
        key = lp / temperature - torch.log(-torch.log(u))
        key = key.masked_fill(~keep, NEG_INF)
        best2 = key.topk(2, 1)
        pred = best2.indices[:, 0]
        clear = (best2.values[:, 0] - best2.values[:, 1]) > 1e-5
        assert bool(keep.gather(1, tokens.long()[:, None]).all()), 'drawn outside the kept set'
        assert torch.equal(tokens.long()[clear], pred[clear]), (step, tokens.tolist(), pred.tolist())
        e = float((picked.double() - lp.gather(1, tokens.long()[:, None])[:, 0]).abs().max())
        _note('picked_lp (samplers)', e)
        assert e < TOL_ROW
        checked += int(clear.sum())
        total += rows
    assert checked >= 0.95 * total


@gpu
def test_draws_do_not_depend_on_the_number_of_rows(L):
    """One row, 50 rows and 1280 rows of one launch: the rows they share draw the same words (the noise is a function of (word, row,
    step, seed) only)."""
    V1 = 100001
    g = torch.Generator(device='cuda').manual_seed(4)
    x = torch.randn(1280, V1, generator=g, device='cuda') * 3
    for select, top in ((MULTINOMIAL, 0.0), (TOPK, 50.0), (NUCLEUS, 0.9)):
        few, _, _, _ = run_select(L, x[:1], select, top, 1.1, seed=9, step=3)
        mid, _, _, _ = run_select(L, x[:50], select, top, 1.1, seed=9, step=3)
        many, _, _, _ = run_select(L, x, select, top, 1.1, seed=9, step=3)
        assert torch.equal(few, many[:1]) and torch.equal(mid, many[:50])
        assert len(set(many.tolist())) > 1000


def _pooled_chi2(counts, q, n, min_expected=20.0):
    order = np.argsort(-q, kind='stable')
    e_bins, o_bins, e, o = [], [], 0.0, 0.0
    for i in order:
        e += q[i] * n
        o += counts[i]
        if e >= min_expected:
            e_bins.append(e)
            o_bins.append(o)
            e, o = 0.0, 0.0
    if e > 0 and e_bins:
        e_bins[-1] += e
        o_bins[-1] += o
    e_bins, o_bins = np.array(e_bins), np.array(o_bins)
    return float(((o_bins - e_bins) ** 2 / e_bins).sum()), len(e_bins) - 1


@gpu
@pytest.mark.parametrize('V1', [60001, 409600])
def test_multinomial_distribution(L, V1):
    """102 400 draws of one Zipf row (2048 rows x 50 launches, different step and seed) against softmax in float64: chi-square over
    the words, tail pooled to expected counts >= 20, and over the CTA slices of the cluster."""
    temperature = 1.25
    row = zipf_rows(V1, (1.25,), seed=V1 + 1)[0]
    q = torch.softmax(ref_logp(row[None])[0] / temperature, 0).numpy()
    x = row.cuda()[None].expand(2048, V1)
    counts = np.zeros(V1)
    launches = 50
    for i in range(launches):
        tokens, _, _, _ = run_select(L, x, MULTINOMIAL, 0.0, temperature, seed=1000 + i // 10, step=i)
        counts += np.bincount(tokens.cpu().numpy(), minlength=V1)
    n = 2048 * launches
    chi2, dof = _pooled_chi2(counts, q, n)
    print('\n[large vocab step] multinomial V1=%d: chi2 %.1f, dof %d' % (V1, chi2, dof))
    assert dof > 50 and chi2 < dof + 6 * (2 * dof) ** 0.5, (chi2, dof)
    o = np.array([counts[lo:hi].sum() for lo, hi in slices(V1)])
    e = np.array([q[lo:hi].sum() for lo, hi in slices(V1)]) * n
    c2 = float(((o - e) ** 2 / e).sum())
    assert c2 < (len(o) - 1) + 6 * (2 * (len(o) - 1)) ** 0.5, (o, e)


@gpu
@pytest.mark.parametrize('select', [GREEDY, MULTINOMIAL])
def test_finished_rows_emit_pad(L, select):
    V1 = 60001
    x = torch.randn(12, V1, generator=torch.Generator().manual_seed(9)) * 4
    x[5, 0] = 50.0                                                  # a live row that ends now
    x = x.cuda()
    lp = ref_logp(x)
    flags = torch.ones(12, dtype=torch.int32)
    flags[[1, 4, 11]] = 0
    unfinished = flags.cuda()
    tokens, picked, row, _ = run_select(L, x, select, unfinished=unfinished, first_step=0)
    tokens, picked, row = tokens.cpu(), picked.cpu(), row.cpu()
    done = flags == 0
    assert bool((tokens[done] == 0).all()) and bool((picked[done] == 0).all()) and bool((row[done] == 0).all())
    assert row_error(row[~done], lp.cpu()[~done]) < TOL_ROW
    assert int(tokens[5]) == 0
    assert unfinished.cpu().tolist() == [int(f and t != 0) for f, t in zip(flags.tolist(), tokens.tolist())]
    if select == GREEDY:
        assert tokens[~done].tolist() == ref_order(x, 1)[:, 0].cpu()[~done].tolist()


# ---------------------------------------------------------------------------------------------------------------------------------
# D. the limit
# ---------------------------------------------------------------------------------------------------------------------------------
@gpu
def test_rows_above_the_limit_are_refused_before_any_launch(L):
    V1 = MAX_ROW + 1
    x = torch.randn(2, V1, device='cuda')
    before = x.clone()
    tokens = torch.full((2,), -7, dtype=torch.int32, device='cuda')
    picked = torch.full((2,), 7.0, device='cuda')
    rc = L.load().capb200_vocab_select(L.ptr(x), V1, 2, V1, GREEDY, 0.0, 1.0, 1, 0, None, 1, L.ptr(tokens), L.ptr(picked), L.current_stream())
    torch.cuda.synchronize()
    assert rc != 0 and b'409600' in L.load().capb200_last_error()
    assert torch.equal(x, before) and bool((tokens == -7).all()) and bool((picked == 7.0).all())
    tv = torch.full((2, 5), 7.0, device='cuda')
    ti = torch.full((2, 5), -7, dtype=torch.int32, device='cuda')
    rc = L.load().capb200_log_softmax_topk(L.ptr(x), V1, 2, V1, 0, 5, L.ptr(tv), L.ptr(ti), L.current_stream())
    torch.cuda.synchronize()
    assert rc != 0 and b'409600' in L.load().capb200_last_error()
    assert torch.equal(x, before) and bool((tv == 7.0).all())
    # the largest supported row runs, and beam search's statistics kernel has no such limit
    tokens, _, _, _ = run_select(L, x[:, :MAX_ROW], GREEDY)
    assert torch.equal(tokens.long(), ref_order(x[:, :MAX_ROW], 1)[:, 0])
    stats = torch.empty(2, 2, device='cuda')
    L.check(L.load().capb200_vocab_stats_topk(L.ptr(x), V1, 2, V1, 1, 5, L.ptr(stats), L.ptr(tv), L.ptr(ti), L.current_stream()), 'stats')
    torch.cuda.synchronize()
    assert torch.equal(ti.long(), ref_order(x, 5))
