"""The vocabulary-step kernels (csrc/vocab.cu) against float64 at real vocabulary size, through the operator-level entry points
capb200_vocab_stats_topk (beam search's statistics / top-k kernel, its rescan branch and its non-vector fallback) and
capb200_vocab_select (greedy, multinomial, top-k and nucleus choice of _sample).

References are a few lines of torch float64 below: the row maximum and log(sum(exp(x - max))), a stable descending sort of the fp32
inputs (value descending, index ascending), and the kept sets of sample_next_word (CaptionModel.py:375-406).  One CPU test checks
those helpers against brute-force loops, so a wrong reference cannot hide a wrong kernel.

The statistics kernel has two forms: the 128-thread single-pass kernel for 16-byte aligned rows and the two-pass scalar kernel for the
rest (a width or pitch that is not a multiple of four, a misaligned base); the `stats` tests reach both.

Largest errors against float64 observed on one H100 (80 GB HBM3, 700 W): log-sum-exp 4.8e-7 with the default single-pass kernel and
6.0e-7 with the two-pass forms, candidate log-probs 1.4e-6, the sampling kernel's stored row 1.2e-6, its picked log-prob 1.2e-6; the
bars below (5e-6, and 1e-5 for the sampling kernel) leave a factor of four.
"""
import numpy as np
import pytest
import torch

SENTINEL = 0x7fffffff
NEG_INF = float('-inf')
HAS_GPU = torch.cuda.is_available()
TOL = 5e-6                      # log-sum-exp and candidate log-probs against float64
ULP = 2.0 ** -23                # plus the roundings of the fp32 result itself where its magnitude is large

OBSERVED = {}                   # name -> largest error seen in this process (printed at teardown; visible with -s)


def gpu(fn):
    return pytest.mark.gpu(pytest.mark.skipif(not HAS_GPU, reason='needs a CUDA device')(fn))


def _note(name, v):
    OBSERVED[name] = max(OBSERVED.get(name, 0.0), float(v))


@pytest.fixture(scope='module')
def L():
    import imagecaptioning.pytorch_b200 as b200
    yield b200._lib
    if OBSERVED:
        print('\n[vocab step] largest errors against float64: ' + ', '.join('%s %.3g' % kv for kv in sorted(OBSERVED.items())))


# ---------------------------------------------------------------------------------------------------------------------------------
# float64 references
# ---------------------------------------------------------------------------------------------------------------------------------
def ref_stats(x):
    """Row maximum and log(sum(exp(x - max))) in float64."""
    xd = x.double()
    mx = xd.max(1, keepdim=True).values
    lse = (xd - mx).exp().sum(1, keepdim=True).log()
    return mx[:, 0], lse[:, 0]


def ref_logp(x, twice=False):
    xd = x.double()
    lp = xd - torch.logsumexp(xd, -1, keepdim=True)
    if twice:
        lp = lp - torch.logsumexp(lp, -1, keepdim=True)
    return lp


def ref_order(x, k):
    """Columns of the k largest entries of each row: value descending, lowest column first on ties (a stable sort of the fp32 inputs)."""
    return torch.sort(x, dim=-1, descending=True, stable=True).indices[..., :k]


def kept_topk(x, k):
    """top-k sampling (CaptionModel.py:398-402) keeps the k most likely words; every word tied with the k-th is kept (torch.topk
    would pick arbitrarily among them)."""
    if k >= x.numel():
        return torch.ones_like(x, dtype=torch.bool)
    return x >= torch.sort(x, descending=True).values[k - 1]


def kept_nucleus(x, p, temperature):
    """Nucleus sampling (CaptionModel.py:388-397): a word is kept iff the mass, under softmax(logp / T), of the strictly more likely
    words is below p -- the reference's shifted cumulative-sum mask, with tied words sharing one fate."""
    q = torch.softmax(ref_logp(x) / temperature, -1)
    xs, order = torch.sort(x, descending=True, stable=True)
    cum = torch.cat([torch.zeros(1, dtype=torch.float64), q[order].cumsum(0)])
    n_above = torch.searchsorted(-xs, -xs, right=False)            # words strictly more likely than each sorted word
    keep = torch.zeros_like(x, dtype=torch.bool)
    keep[order] = cum[n_above] < p
    return keep, cum[n_above][torch.argsort(order)]


def test_reference_helpers_against_brute_force():
    g = torch.Generator().manual_seed(50)
    x = torch.randn(50, generator=g) * 2
    x[[7, 19]] = x[3].item()                                           # one three-way tie in the middle of the order
    xs = x.tolist()
    # stable top-k by selection
    taken, order = set(), []
    for _ in range(50):
        best = None
        for i, v in enumerate(xs):
            if i not in taken and (best is None or v > xs[best]):
                best = i
        taken.add(best)
        order.append(best)
    assert ref_order(x, 50).tolist() == order
    assert ref_order(x.unsqueeze(0), 5)[0].tolist() == order[:5]
    # statistics and log-probs
    mx, lse = ref_stats(x.unsqueeze(0))
    m = max(xs)
    s = sum(np.exp(np.float64(v) - m) for v in xs)
    assert float(mx) == m and abs(float(lse) - np.log(s)) < 1e-14
    lp = [np.float64(v) - m - np.log(s) for v in xs]
    assert np.abs(ref_logp(x).numpy() - np.array(lp)).max() < 1e-13
    assert np.abs(ref_logp(x, twice=True).numpy() - np.array(lp)).max() < 1e-13
    rank_of_tie = order.index(3)
    for temperature in (0.5, 1.0, 2.0):
        q = np.exp(np.array(lp) / temperature)
        q /= q.sum()
        for k in sorted({1, 5, 17, 50, 60, rank_of_tie + 1, rank_of_tie + 2, rank_of_tie + 3}):
            keep = [False] * 50
            for i in order[:k]:
                keep[i] = True
            mine = kept_topk(x, k).tolist()
            if rank_of_tie < k <= rank_of_tie + 2:                 # the cut falls inside the tie: all three tied words are kept
                assert sum(mine) == rank_of_tie + 3 and all(m_ or not k_ for m_, k_ in zip(mine, keep))
            else:
                assert mine == keep
        for p in (1e-6, 0.3, 0.6, 0.9, 1.0):
            # the reference: sort, cumulative sum, keep while the sum is below p, shifted by one so the first word always stays
            csum, keep = 0.0, [False] * 50
            for j, i in enumerate(order):
                keep[i] = (j == 0) or (csum < p)
                csum += q[i]
            mine, mass = kept_nucleus(x, p, temperature)
            differs = [i for i in range(50) if mine[i] != keep[i]]
            assert set(differs) <= {3, 7, 19}                     # only the tie can differ: the reference splits it, this keeps or drops it whole
            assert abs(float(mass[order[1]]) - q[order[0]]) < 1e-14


# ---------------------------------------------------------------------------------------------------------------------------------
# launchers
# ---------------------------------------------------------------------------------------------------------------------------------
LAYOUTS = ['dense', 'pitch4', 'pitch1', 'offset1']       # ld == V1 | ld = V1 + 4 | ld = V1 + 1 (scalar fallback) | base + 1 float (fallback)


def place(x, layout):
    """The rows of x on the device in one of the layouts; every float around them holds +1e30, so a kernel that reads outside a row
    finds a wrong maximum.  Returns (owning buffer, [rows, V1] view, pitch)."""
    rows, V1 = x.shape
    if layout == 'dense':
        buf = x.to('cuda', copy=True).contiguous()                  # never the caller's tensor: the sampling kernel rewrites its rows
        return buf, buf, V1
    if layout in ('pitch4', 'pitch1'):
        ld = V1 + (4 if layout == 'pitch4' else 1)
        buf = torch.full((rows, ld), 1e30, device='cuda')
        buf[:, :V1] = x.cuda()
        return buf, buf[:, :V1], ld
    buf = torch.full((rows * V1 + 4,), 1e30, device='cuda')
    view = buf[1:1 + rows * V1].view(rows, V1)
    view.copy_(x.cuda())
    return buf, view, V1


def run_stats(L, x, k, twice=0, layout='dense'):
    rows, V1 = x.shape
    buf, view, ld = place(x, layout)
    before = buf.clone()
    stats = torch.full((rows, 2), 7.0, device='cuda')
    top_val = torch.full((rows, k), 7.0, device='cuda')
    top_idx = torch.full((rows, k), -7, dtype=torch.int32, device='cuda')
    L.check(L.load().capb200_vocab_stats_topk(L.ptr(view), ld, rows, V1, twice, k, L.ptr(stats), L.ptr(top_val), L.ptr(top_idx), L.current_stream()),
            'vocab_stats_topk')
    torch.cuda.synchronize()
    assert torch.equal(buf, before), 'the statistics kernel must leave the logits (and everything around them) untouched'
    return stats.cpu(), top_val.cpu(), top_idx.cpu()


def check_stats(L, x, k, twice=0, layout='dense', tag='stats'):
    """One launch of the statistics / top-k kernel against float64: indices equal the stable sort bit for bit on every row, the maximum
    exactly, log-sum-exp and candidate log-probs within TOL.  Past a row's last entry above -inf the kernel reports value -inf with the
    sentinel index, or with a column that holds -inf (a thread that rescans its words lists them); never another index >= V1."""
    rows, V1 = x.shape
    stats, top_val, top_idx = run_stats(L, x, k, twice, layout)
    mx, lse = ref_stats(x)
    assert torch.equal(stats[:, 0].double(), mx), (tag, 'row max')
    err = (stats[:, 1].double() - lse).abs().max()
    _note('stats lse', err)
    assert err <= TOL, (tag, 'log-sum-exp', float(err))
    order = ref_order(x, k)
    n_finite = (x > NEG_INF).sum(1)
    lp = ref_logp(x, bool(twice))
    for r in range(rows):
        n = min(int(n_finite[r]), k)
        assert top_idx[r, :n].tolist() == order[r, :n].tolist(), (tag, layout, 'row', r, top_idx[r].tolist(), order[r].tolist())
        ref_v = lp[r, order[r, :n]]
        e = (top_val[r, :n].double() - ref_v).abs() - 4 * ULP * ref_v.abs()
        if n:
            _note('top_val', (top_val[r, :n].double() - ref_v).abs().max() if float(ref_v.abs().max()) < 100 else 0.0)
            assert float(e.max()) <= TOL, (tag, layout, 'row', r, float(e.max()))
        for j in range(n, k):
            i = int(top_idx[r, j])
            assert float(top_val[r, j]) == NEG_INF and (i == SENTINEL or (0 <= i < V1 and float(x[r, i]) == NEG_INF)), (tag, r, j, i)


def owned(c, nthreads, V1, vector):
    """Columns thread c of an nthreads-wide CTA visits: whole float4 groups c, c + nthreads, ... or single columns c, c + nthreads, ..."""
    if vector:
        return [4 * g + u for g in range(c, V1 // 4, nthreads) for u in range(4) if 4 * g + u < V1]
    return list(range(c, V1, nthreads))


def plant(row, cols, rng, base=10.0, step=0.5):
    """Puts distinct large values on `cols` in a random value order (the best need not be the first visited)."""
    vals = base + step * rng.permutation(len(cols))
    row[torch.tensor(cols)] = torch.tensor(vals, dtype=torch.float32)


def adversarial_rows(V1, k, seed):
    """Rows whose k largest values all belong to one thread (or alternate between two) of each kernel form: the 128-thread float4
    kernel (four loads in flight, then a tail loop), the 256-thread float4 forms and the 256-thread scalar fallback; and rows whose
    k largest are the last k columns."""
    rng = np.random.RandomState(seed)
    g = torch.Generator().manual_seed(seed)
    rows = []
    for nthreads, vector in ((128, True), (256, True), (256, False)):
        for c in (0, 1, 31, 67, nthreads - 1):
            mine = owned(c, nthreads, V1, vector)
            if len(mine) < k:
                continue
            # always the first float4 / first column, two more of the same float4, and the last one visited; the rest at random
            forced = [mine[0], mine[-1]] + ([mine[1], mine[3]] if vector else [mine[1], mine[len(mine) // 2]])
            rest = [m for m in mine if m not in forced]
            cols = (forced + list(rng.permutation(rest)))[:k]
            row = torch.randn(V1, generator=g)
            plant(row, cols, rng)
            rows.append(row)
            # two threads alternately
            other = owned((c + 5) % nthreads, nthreads, V1, vector)
            if len(other) >= k:
                both = [m for pair in zip(mine, other) for m in pair][:k]
                row = torch.randn(V1, generator=g)
                row[torch.tensor(both)] = torch.tensor(10.0 + 0.5 * np.arange(len(both))[::-1].copy(), dtype=torch.float32)
                rows.append(row)
    if V1 >= k:
        row = torch.randn(V1, generator=g)
        plant(row, list(range(V1 - k, V1)), rng)
        rows.append(row)
    return torch.stack(rows)


KS = [1, 2, 3, 5, 10, 16]


# ---------------------------------------------------------------------------------------------------------------------------------
# A. statistics / top-k kernel
# ---------------------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('k', [1, 5, 16])
@pytest.mark.parametrize('V1,rows', [(9488, 1), (9488, 17), (9488, 1280), (9487, 17), (9487, 1280), (9490, 17), (4, 17), (8, 17), (100, 17),
                                     (512, 17), (513, 17), (2048, 17), (51204, 1), (51204, 17)])
def test_stats_shapes(L, V1, rows, k):
    g = torch.Generator().manual_seed(V1 * 31 + rows + k)
    x = torch.randn(rows, V1, generator=g) * 4
    for twice in (0, 1):
        check_stats(L, x, k, twice, 'dense', tag=('shape', V1, rows, k, twice))


@gpu
@pytest.mark.parametrize('layout', ['pitch4', 'pitch1', 'offset1'])
@pytest.mark.parametrize('V1', [9488, 9487, 512, 8])
def test_stats_pitched_and_misaligned_slabs(L, V1, layout):
    g = torch.Generator().manual_seed(V1 + len(layout))
    x = torch.randn(17, V1, generator=g) * 4
    for k in (1, 5, 16):
        check_stats(L, x, k, 1, layout, tag=('layout', V1, layout, k))


@gpu
@pytest.mark.parametrize('layout', LAYOUTS)
@pytest.mark.parametrize('k', KS)
@pytest.mark.parametrize('V1', [9488, 9487])
def test_stats_topk_owned_by_one_thread(L, V1, k, layout):
    """With k = 16 on one thread the rescan branch runs 14 times in a row; random rows reach it about once in two thousand."""
    x = adversarial_rows(V1, k, seed=V1 + k)
    check_stats(L, x, k, 1, layout, tag=('owned', V1, k))


@gpu
@pytest.mark.parametrize('layout', ['dense', 'pitch1'])
@pytest.mark.parametrize('k', KS)
@pytest.mark.parametrize('V1', [9488, 9487, 100])
def test_stats_ties(L, V1, k, layout):
    g = torch.Generator().manual_seed(V1 + k)
    rng = np.random.RandomState(V1 + k)
    rows = [torch.zeros(V1), torch.full((V1,), -3.25)]                               # all equal: columns 0 .. k-1
    row = torch.randn(V1, generator=g)
    row[torch.from_numpy(rng.choice(V1, 2 * k, replace=False))] = 9.0               # the top value 2k times, spread over threads
    rows.append(row)
    for nthreads, vector in ((128, True), (256, False)):                            # ... and 2k times inside one thread
        mine = owned(3, nthreads, V1, vector)
        if len(mine) >= 2 * k:
            row = torch.randn(V1, generator=g)
            row[torch.tensor(mine[:k] + mine[-k:])] = 9.0
            rows.append(row)
    row = torch.randn(V1, generator=g)                                              # a tie that straddles the k-th place
    cols = rng.choice(V1, k + 3, replace=False)
    row[torch.from_numpy(cols[:max(k - 2, 0)])] = 12.0 + torch.arange(max(k - 2, 0), dtype=torch.float32)
    row[torch.from_numpy(cols[max(k - 2, 0):])] = 9.0
    rows.append(row)
    row = torch.randn(V1, generator=g)                                              # ties inside one float4, and the next float4 of that thread
    row[40:44] = 9.0
    row[40 + 512:44 + 512] = 9.0
    rows.append(row)
    check_stats(L, torch.stack(rows), k, 1, layout, tag=('ties', V1, k))


@gpu
@pytest.mark.parametrize('layout', ['dense', 'pitch1'])
@pytest.mark.parametrize('V1', [9488, 9487])
def test_stats_value_ranges(L, V1, layout):
    g = torch.Generator().manual_seed(V1)
    base = torch.randn(6, V1, generator=g)
    rows = [base[0], base[0] * 20, base[0] * 1e3,                                   # one term dominates; everything else flushes to zero
            base[1] * 4 + 3e4, base[1] * 4 - 3e4,                                   # a large common offset
            (torch.randperm(V1, generator=g).float() * 2.0 ** -149),                # denormal spacing
            torch.arange(V1, dtype=torch.float32) * 1e-3,                           # the maximum is the last element: every step rescales
            -torch.arange(V1, dtype=torch.float32) * 1e-3,                          # ... and the first
            torch.arange(V1, dtype=torch.float32) * 0.05]
    row = base[2].clone() * 4                                                       # -inf in scattered columns
    row[torch.randperm(V1, generator=g)[:V1 // 3]] = NEG_INF
    rows.append(row)
    row = base[3].clone() * 4                                                       # ... in whole float4 groups, the first ones of many threads included
    row[:1024] = NEG_INF
    row[4000:4400] = NEG_INF
    rows.append(row)
    for nthreads, vector in ((128, True), (256, True), (256, False)):               # ... in every column one thread owns
        row = base[4].clone() * 4
        row[torch.tensor(owned(5, nthreads, V1, vector))] = NEG_INF
        rows.append(row)
        row = base[5].clone() * 4                                                   # ... in all but that thread's last column
        row[torch.tensor(owned(5, nthreads, V1, vector)[:-1])] = NEG_INF
        rows.append(row)
    x = torch.stack(rows)
    for k in (1, 5, 16):
        for twice in (0, 1):
            check_stats(L, x, k, twice, layout, tag=('values', V1, k, twice))


@gpu
@pytest.mark.parametrize('layout', ['dense', 'pitch1'])
def test_stats_fewer_candidates_than_k(L, layout):
    """Rows with fewer than k entries above -inf, and V1 = 4 with k = 5.  The missing places carry -inf and the sentinel index (or a
    column holding -inf), never another index >= V1.  The beam kernels cannot index with the sentinel: every decode entry point
    requires beam_size <= V+1, so the candidate list of a row always holds beam_size real words; a list widened for decode edits
    (k_in > V+1) is cut back to beam_size by beam_edit_kernel, which only compares the index and prefers real words on ties."""
    for V1, k in ((4, 5), (4, 16), (8, 10), (9488, 5), (9488, 16)):
        g = torch.Generator().manual_seed(V1 + k)
        x = torch.full((6, V1), NEG_INF)
        for r, n in enumerate((1, 2, 3, min(k - 1, V1), min(k, V1), V1)):
            cols = torch.randperm(V1, generator=g)[:n]
            x[r, cols] = torch.randn(n, generator=g)
        check_stats(L, x, k, 1, layout, tag=('few', V1, k))
        _, top_val, top_idx = run_stats(L, x, k, 0, layout)
        assert int(top_idx[0, 1]) == SENTINEL and float(top_val[0, 1]) == NEG_INF      # a single-entry row never rescans: the plain sentinel


@gpu
def test_stats_beam_width_bounds(L):
    x = torch.randn(3, 9488, generator=torch.Generator().manual_seed(1))
    check_stats(L, x, 16, 1, 'dense', tag='k16')
    xd = x.cuda()
    stats = torch.full((3, 2), 7.0, device='cuda')
    top_val = torch.full((3, 17), 7.0, device='cuda')
    top_idx = torch.full((3, 17), -7, dtype=torch.int32, device='cuda')
    rc = L.load().capb200_vocab_stats_topk(L.ptr(xd), 9488, 3, 9488, 1, 17, L.ptr(stats), L.ptr(top_val), L.ptr(top_idx), L.current_stream())
    torch.cuda.synchronize()
    assert rc != 0 and b'beam size up to 16' in L.load().capb200_last_error()
    assert bool((stats == 7.0).all()) and bool((top_val == 7.0).all()) and bool((top_idx == -7).all())      # nothing was launched
    with pytest.raises(RuntimeError, match='bad argument'):
        L.check(L.load().capb200_vocab_stats_topk(L.ptr(xd), 9488, 3, 9488, 1, 0, L.ptr(stats), L.ptr(top_val), L.ptr(top_idx), L.current_stream()))


# ---------------------------------------------------------------------------------------------------------------------------------
# B. the ways to a top-k agree
# ---------------------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('V1,twice,k', [(9488, 1, 5), (9488, 0, 16), (9487, 1, 10), (1000, 1, 1)])
def test_stats_topk_agrees_with_log_softmax_topk(L, V1, twice, k):
    """capb200_log_softmax_topk ranks on the rounded log-probs, the statistics kernel on the raw logits: same values, and the same
    columns wherever float64 separates a candidate from the next by more than 1e-5."""
    g = torch.Generator().manual_seed(V1 + k)
    x = torch.cat([torch.randn(17, V1, generator=g) * 4, adversarial_rows(V1, k, seed=k)])
    rows = x.shape[0]
    _, sv, si = run_stats(L, x, k, twice)
    xd = x.cuda()
    tv = torch.empty(rows, k, device='cuda')
    ti = torch.empty(rows, k, dtype=torch.int32, device='cuda')
    L.check(L.load().capb200_log_softmax_topk(L.ptr(xd), V1, rows, V1, twice, k, L.ptr(tv), L.ptr(ti), L.current_stream()), 'log_softmax_topk')
    torch.cuda.synchronize()
    tv, ti = tv.cpu(), ti.cpu()
    lp = ref_logp(x, bool(twice))
    assert float((xd.cpu().double() - lp).abs().max()) < 1e-5
    assert float((tv.double() - sv.double()).abs().max()) <= TOL
    sorted_lp = torch.sort(lp, 1, descending=True).values[:, :k + 1]
    clear = (sorted_lp[:, :-1] - sorted_lp[:, 1:]) > 1e-5          # place j is decided iff it is clear of place j + 1 ...
    clear[:, 1:] &= clear[:, :-1].clone()                          # ... and of place j - 1
    assert bool(clear.float().mean() > 0.99)
    assert torch.equal(ti[clear], si[clear])


# ---------------------------------------------------------------------------------------------------------------------------------
# C. samplers
# ---------------------------------------------------------------------------------------------------------------------------------
GREEDY, MULTINOMIAL, TOPK, NUCLEUS = 1, 2, 4, 5


def run_select(L, x, select, top=0.0, temperature=1.0, seed=1234, step=0, unfinished=None, first_step=1, layout='dense', keep_row=False):
    """x: [rows, V1] (CPU or device).  Returns tokens, picked log-probs (CPU) and, if keep_row, the rewritten slab with its surroundings."""
    rows, V1 = x.shape
    buf, view, ld = place(x, layout)
    tokens = torch.full((rows,), -7, dtype=torch.int32, device='cuda')
    picked = torch.full((rows,), 7.0, device='cuda')
    L.check(L.load().capb200_vocab_select(L.ptr(view), ld, rows, V1, select, top, temperature, seed, step, L.ptr(unfinished), first_step,
                                          L.ptr(tokens), L.ptr(picked), L.current_stream()), 'vocab_select')
    torch.cuda.synchronize()
    if keep_row:
        return tokens.cpu(), picked.cpu(), buf.cpu(), view.cpu()
    return tokens.cpu(), picked.cpu()


@gpu
@pytest.mark.parametrize('layout', ['dense', 'pitch4', 'pitch1'])
@pytest.mark.parametrize('V1', [9488, 9487])
def test_greedy_is_the_stable_argmax(L, V1, layout):
    g = torch.Generator().manual_seed(V1)
    x = torch.randn(40, V1, generator=g) * 4
    x[1] *= 5
    x[2, [77, 5000, 9000]] = 30.0                                   # tied maxima: the lowest column wins
    x[3] = 0.0
    x[4, V1 - 1] = 40.0
    x[5, [V1 - 1, V1 - 2]] = 40.0
    tokens, picked, buf, row = run_select(L, x, GREEDY, layout=layout, keep_row=True)
    lp = ref_logp(x)
    assert tokens.tolist() == ref_order(x, 1)[:, 0].tolist()
    e_pick = (picked.double() - lp.gather(1, tokens.long().unsqueeze(1))[:, 0]).abs().max()
    e_row = ((row.double() - lp).abs() - 2 * ULP * lp.abs()).max()  # row 1 reaches -150, where one fp32 ulp is 1.5e-5
    _note('picked_lp', e_pick)
    _note('log-softmax row', (row.double() - lp).abs()[lp > -16].max())
    assert float(e_pick) < 1e-5 and float(e_row) < 1e-5
    if layout != 'dense':
        assert bool((buf[:, V1:] == 1e30).all())                    # the pitch columns are neither read nor written


def zipf_rows(V1, exponents, seed):
    """Rows whose sorted log-probs fall like -s * log(rank): neighbours in the order are s / rank apart, so the 50 best are separated by
    more than 1e-2.  Words are scattered over the columns."""
    g = torch.Generator().manual_seed(seed)
    rows = []
    for s in exponents:
        row = torch.empty(V1)
        row[torch.randperm(V1, generator=g)] = -s * torch.log(torch.arange(1, V1 + 1, dtype=torch.float64)).float()
        rows.append(row + 3.0)
    return torch.stack(rows)


KEPT_EXPONENTS = (2.4, 3.0, 3.4, 4.0)
N_ROWS, N_STEPS = 2048, 10                       # 20 480 draws per setting; a slab of 2048 rows is 78 MB


def _draw(L, base, select, top, temperature, seed=99, steps=N_STEPS, rows=N_ROWS):
    """rows x steps draws; row r holds base[r % len(base)].  Returns tokens [steps, rows]."""
    x = base.cuda()[torch.arange(rows, device='cuda') % base.shape[0]]
    out = []
    for step in range(steps):
        tokens, _ = run_select(L, x, select, top, temperature, seed=seed, step=step)
        out.append(tokens)
    return torch.stack(out).long()


def _check_kept(tokens, base, keep, q):
    """No draw outside the kept set; and every kept word expected at least 20 times was drawn (the set is not too small either)."""
    kinds = torch.arange(tokens.shape[1]) % base.shape[0]
    for b in range(base.shape[0]):
        t = tokens[:, kinds == b].reshape(-1)
        counts = torch.bincount(t, minlength=base.shape[1])
        assert int(counts[~keep[b]].sum()) == 0, ('drawn outside the kept set', b, torch.nonzero(counts * ~keep[b])[:5].tolist())
        qq = q[b] * keep[b]
        expected = qq / qq.sum() * t.numel()
        assert bool((counts[expected >= 20] > 0).all()), ('a kept word was never drawn', b)


@gpu
@pytest.mark.parametrize('temperature', [0.5, 1.0, 2.0])
@pytest.mark.parametrize('k', [1, 5, 50, 9488])
@pytest.mark.parametrize('V1', [9488, 9487])
def test_topk_sampler_kept_set(L, V1, k, temperature):
    base = zipf_rows(V1, KEPT_EXPONENTS, seed=V1)
    lp = ref_logp(base)
    srt = torch.sort(lp, 1, descending=True).values
    if k < V1:
        assert float((srt[:, k - 1] - srt[:, k]).min()) >= 1e-3       # the threshold word is clear of its neighbour
    keep = torch.stack([kept_topk(r, k) for r in base])
    q = torch.softmax(lp / temperature, 1)
    tokens = _draw(L, base, TOPK, float(k), temperature)
    _check_kept(tokens, base, keep, q)
    if k == 1:                                                      # top-1 is greedy on every draw
        assert bool((tokens == ref_order(base, 1)[:, 0][torch.arange(N_ROWS) % len(base)]).all())
    if k >= V1:                                                     # nothing is cut: the same noise picks the same words as the plain multinomial
        assert torch.equal(tokens[:2], _draw(L, base, MULTINOMIAL, 0.0, temperature, steps=2))


@gpu
@pytest.mark.parametrize('temperature', [0.5, 1.0, 2.0])
@pytest.mark.parametrize('p', [1e-6, 0.3, 0.9, 1.0])
@pytest.mark.parametrize('V1', [9488, 9487])
def test_nucleus_sampler_kept_set(L, V1, p, temperature):
    base = zipf_rows(V1, KEPT_EXPONENTS, seed=V1)
    q = torch.softmax(ref_logp(base) / temperature, 1)
    keep, mass = zip(*[kept_nucleus(r, p, temperature) for r in base])
    keep, mass = torch.stack(keep), torch.stack(mass)
    if p < 1.0:
        assert float((mass[mass > 0] - p).abs().min()) > 5e-6       # no word sits on the threshold: fp32 mass sums cannot change the set
    tokens = _draw(L, base, NUCLEUS, p, temperature)
    _check_kept(tokens, base, keep, q)
    if p == 1e-6:                                                   # only the most likely word survives: greedy on every draw
        assert bool((tokens == ref_order(base, 1)[:, 0][torch.arange(N_ROWS) % len(base)]).all())


@gpu
@pytest.mark.parametrize('V1', [9488, 9487])
def test_truncated_samplers_keep_every_word_tied_at_the_threshold(L, V1):
    """An exact tie at the cut: the kernel keeps all tied words (a deviation from torch.topk's arbitrary pick, CaptionModel.py:399).
    And a threshold one ulp wide: with one dominant word at 0 and the others below -200 the log-softmax returns the logits bit for
    bit, so the 5th and 6th words can be made adjacent floats; top-5 keeps exactly five."""
    g = torch.Generator().manual_seed(V1)
    row = torch.randn(V1, generator=g) * 0.5 - 6.0
    tied = torch.randperm(V1, generator=g)[:8]
    row[tied[:3]] = torch.tensor([6.0, 5.5, 5.0])
    row[tied[3:]] = 4.0                                             # places 4..8 are tied: top-5 keeps all eight
    keep = kept_topk(row, 5)
    assert int(keep.sum()) == 8
    tokens = _draw(L, row.unsqueeze(0), TOPK, 5.0, 2.0, steps=4)
    counts = torch.bincount(tokens.reshape(-1), minlength=V1)
    assert int(counts[~keep].sum()) == 0 and bool((counts[keep] > 0).all())
    keep_p, _ = kept_nucleus(row, 0.75, 1.0)                        # the tie straddles p = 0.75 as well
    assert int(keep_p.sum()) == 8
    tokens = _draw(L, row.unsqueeze(0), NUCLEUS, 0.75, 1.0, steps=4)
    counts = torch.bincount(tokens.reshape(-1), minlength=V1)
    assert int(counts[~keep_p].sum()) == 0 and bool((counts[keep_p] > 0).all())

    row = -300.0 - torch.rand(V1, generator=g) * 100
    cols = torch.randperm(V1, generator=g)[:6]
    fifth = torch.tensor(-205.0)
    sixth = torch.nextafter(fifth, torch.tensor(NEG_INF))
    row[cols] = torch.stack([torch.tensor(0.0), torch.tensor(-201.0), torch.tensor(-202.0), torch.tensor(-203.0), fifth, sixth])
    _, _, _, written = run_select(L, row.unsqueeze(0), GREEDY, keep_row=True)
    assert torch.equal(written[0], row)                             # the premise: this row's log-softmax is the row itself
    tokens = _draw(L, row.unsqueeze(0), TOPK, 5.0, 200.0, steps=4)
    counts = torch.bincount(tokens.reshape(-1), minlength=V1)
    assert set(torch.nonzero(counts)[:, 0].tolist()) == set(cols[:5].tolist())


def _pooled_chi2(counts, q, n, min_expected=20.0):
    """Chi-square of counts against n * q with the words pooled, most likely first, into bins of expected count >= min_expected."""
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


def _chi2_bound(dof):
    return dof + 6 * (2 * dof) ** 0.5


@gpu
@pytest.mark.parametrize('shape', ['zipf', 'flat'])
@pytest.mark.parametrize('V1', [9488, 9487])
def test_multinomial_distribution_at_vocabulary_size(L, V1, shape):
    """102 400 draws (2048 rows x 50 launches with different step and seed) of one row against softmax in float64: chi-square over the
    words (tail pooled to expected counts >= 20), and over the thread slots word % 256 and word % 1024, which is what a mistake in
    the Philox counter layout or in a strided loop would skew.  Fixed seeds: the test is deterministic."""
    temperature = 1.0 if shape == 'flat' else 1.25
    if shape == 'zipf':
        row = zipf_rows(V1, (1.25,), seed=V1 + 1)[0]                # softmax(logp / 1.25): Zipf with exponent 1
    else:
        row = torch.randn(V1, generator=torch.Generator().manual_seed(V1)) * 0.1
    q = torch.softmax(ref_logp(row) / temperature, 0).numpy()
    x = row.cuda().unsqueeze(0).expand(N_ROWS, V1)
    counts = np.zeros(V1)
    launches = 50
    for i in range(launches):
        tokens, _ = run_select(L, x, MULTINOMIAL, 0.0, temperature, seed=1000 + i // 10, step=i)
        counts += np.bincount(tokens.numpy(), minlength=V1)
    n = N_ROWS * launches
    chi2, dof = _pooled_chi2(counts, q, n)
    print('\n[vocab step] multinomial %s V1=%d: chi2 %.1f, dof %d' % (shape, V1, chi2, dof))
    assert dof > 50 and chi2 < _chi2_bound(dof), (chi2, dof)
    for slots in (256, 1024):
        slot = np.arange(V1) % slots
        o = np.bincount(slot, weights=counts, minlength=slots)
        e = np.bincount(slot, weights=q, minlength=slots) * n
        c2 = float(((o - e) ** 2 / e).sum())
        print('[vocab step] multinomial %s V1=%d: per-slot (%d) chi2 %.1f, dof %d' % (shape, V1, slots, c2, slots - 1))
        assert c2 < _chi2_bound(slots - 1), (slots, c2)


@gpu
@pytest.mark.parametrize('select,top', [(MULTINOMIAL, 0.0), (TOPK, 50.0), (NUCLEUS, 0.9)])
def test_both_block_sizes_draw_the_same_words(L, select, top):
    """Launches of up to 2 * SMs rows run the 1024-thread form of the kernel, larger ones the 256-thread form.  The Gumbel noise is a
    function of (word, row, step, seed) only, so the rows two launches share get the same words."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    V1 = 9488
    g = torch.Generator().manual_seed(int(select))
    x = torch.cat([torch.randn(2048 - 4, V1, generator=g) * 3, zipf_rows(V1, KEPT_EXPONENTS, seed=5)])
    x = x[torch.randperm(2048, generator=g)]
    for step in range(4):
        few, few_lp = run_select(L, x[:2 * sms], select, top, 1.3, seed=7, step=step)
        more, more_lp = run_select(L, x[:2 * sms + 1], select, top, 1.3, seed=7, step=step)
        many, many_lp = run_select(L, x, select, top, 1.3, seed=7, step=step)
        assert torch.equal(few, more[:2 * sms]) and torch.equal(few, many[:2 * sms]) and torch.equal(more, many[:2 * sms + 1])
        assert float((few_lp - many_lp[:2 * sms]).abs().max()) < 4e-6
        lp = ref_logp(x[:2 * sms])
        _note('picked_lp', (few_lp.double() - lp.gather(1, few.long().unsqueeze(1))[:, 0]).abs().max())


@gpu
def test_draws_depend_on_seed_and_step_only(L):
    """A different step or seed changes the draw; the same pair repeats it (a replayed CUDA graph of a training step relies on this)."""
    V1 = 9488
    x = torch.randn(300, V1, generator=torch.Generator().manual_seed(3))
    a, _ = run_select(L, x, MULTINOMIAL, seed=5, step=2)
    b, _ = run_select(L, x, MULTINOMIAL, seed=5, step=2)
    c, _ = run_select(L, x, MULTINOMIAL, seed=5, step=3)
    d, _ = run_select(L, x, MULTINOMIAL, seed=6, step=2)
    e, _ = run_select(L, x, MULTINOMIAL, seed=5, step=2 + 2 ** 32)
    assert torch.equal(a, b)
    for other in (c, d, e):
        assert float((a != other).float().mean()) > 0.9
    assert len(set(a.tolist())) > 200                                # and the rows of one launch draw independently


@gpu
@pytest.mark.parametrize('select', [GREEDY, MULTINOMIAL])
def test_finished_rows_emit_pad(L, select):
    V1 = 9487
    x = torch.randn(12, V1, generator=torch.Generator().manual_seed(9)) * 4
    x[5, 0] = 50.0                                                  # a live row that ends now
    lp = ref_logp(x)
    flags = torch.ones(12, dtype=torch.int32)
    flags[[1, 4, 11]] = 0
    unfinished = flags.cuda()
    tokens, picked, _, row = run_select(L, x, select, unfinished=unfinished, first_step=0, keep_row=True)
    done = flags == 0
    assert bool((tokens[done] == 0).all()) and bool((picked[done] == 0).all()) and bool((row[done] == 0).all())
    assert float((row[~done].double() - lp[~done]).abs().max()) < 1e-5
    assert int(tokens[5]) == 0
    assert unfinished.cpu().tolist() == [int(f and t != 0) for f, t in zip(flags.tolist(), tokens.tolist())]
    # at the first step the flags are ignored (they are rewritten, not read)
    unfinished = flags.cuda()
    tokens, picked, _, row = run_select(L, x, select, unfinished=unfinished, first_step=1, keep_row=True)
    assert float((row.double() - lp).abs().max()) < 1e-5
    assert unfinished.cpu().tolist() == [int(t != 0) for t in tokens.tolist()]
    if select == GREEDY:
        assert tokens.tolist() == ref_order(x, 1)[:, 0].tolist()
