"""GPU parity of the operator-level C-ABI entry points against torch fp64/fp32 CPU references and the golden fixtures."""
import os

import numpy as np
import pytest
import torch

from helpers import LOGP_TOL, co

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def L():
    import imagecaptioning.pytorch_b200 as b200
    return b200._lib


def _linear(L, x, w, b, relu, mode):
    M, K = x.shape
    N = w.shape[0]
    y = torch.empty(M, N, device='cuda')
    L.check(L.load().capb200_linear(L.ptr(x), K, L.ptr(w), K, L.ptr(b), L.ptr(y), N, M, N, K, int(relu), L.OP_MODES[mode], L.current_stream()), 'linear')
    torch.cuda.synchronize()
    return y


@pytest.mark.parametrize('mode', ['simt_fp32', 'tc_f16x3', 'tc_f16x1'])
@pytest.mark.parametrize('shape', [(5, 7, 24), (128, 128, 64), (130, 260, 1000), (1280, 512, 1000), (333, 9488, 1000), (36, 40, 2048)])
def test_linear_matches_fp64(L, mode, shape):
    M, N, K = shape
    g = torch.Generator().manual_seed(M * 7 + N)
    x = torch.randn(M, K, generator=g)
    w = (torch.rand(N, K, generator=g) * 2 - 1) / K ** 0.5
    b = torch.randn(N, generator=g)
    ref = (x.double() @ w.double().t() + b.double())
    y = _linear(L, x.cuda(), w.cuda(), b.cuda(), False, mode).cpu().double()
    err = float((y - ref).abs().max())
    fp32_err = float(((x @ w.t() + b).double() - ref).abs().max())
    # fp32-grade modes must stay within summation-order noise of an fp32 GEMM.  The tensor-core accumulator truncates (round
    # toward zero) once per MMA instruction, so the 3-pass mode gets an explicit budget of one fp32 ulp of the largest
    # output per accumulate (3 * K/16 of them); the single-pass mode is fp16-input grade.
    if mode == 'simt_fp32':
        tol = max(4 * fp32_err, 2e-6)
    elif mode == 'tc_f16x3':
        tol = max(4 * fp32_err, 2e-6) + 3 * (K / 16) * 2.0 ** -24 * float(ref.abs().max())
    else:
        tol = 2e-2
    assert err < tol, (mode, shape, err, fp32_err)
    yr = _linear(L, x.cuda(), w.cuda(), b.cuda(), True, mode).cpu().double()
    assert float((yr - ref.clamp_min(0)).abs().max()) < tol


@pytest.mark.parametrize('mode', ['skinny_tf32x3', 'skinny_fp32'])
@pytest.mark.parametrize('shape', [(5, 7, 24), (50, 4000, 1000), (50, 1000, 4000), (50, 9488, 1000), (360, 1000, 2048), (1000, 1000, 9488), (37, 52, 100)])
def test_skinny_linear_matches_fp64(L, mode, shape):
    """The training step's split-K GEMM: fp32 CUDA-core and 3xTF32 tensor-core variants, fp32-grade against float64; the inputs
    include tiny magnitudes (gradient-like rows) that fp16 planes would flush."""
    M, N, K = shape
    g = torch.Generator().manual_seed(M * 11 + N)
    x = torch.randn(M, K, generator=g)
    x[M // 2:] *= 1e-7
    w = (torch.rand(N, K, generator=g) * 2 - 1) / K ** 0.5
    b = torch.randn(N, generator=g) * 1e-3
    ref = x.double() @ w.double().t() + b.double()
    y = _linear(L, x.cuda(), w.cuda(), b.cuda(), False, mode).cpu().double()
    scale = (x.double().abs() @ w.double().abs().t() + b.double().abs())          # per-element condition scale
    rel = float(((y - ref).abs() / scale).max())
    assert rel < (4e-6 if mode == 'skinny_tf32x3' else 2e-6), (mode, shape, rel)


@pytest.mark.parametrize('shape', [(50, 4096, 3072), (50, 9488, 1024), (50, 1000, 4000), (12, 41, 48), (64, 256, 96), (200, 520, 1000), (360, 3072, 1024),
                                   (1000, 1024, 9488), (257, 130, 36)])
def test_tf32x3_tcgen05_linear_matches_fp64(L, shape):
    """The training steps' wgmma tf32 kernel (gemm_tf32.cu: raw fp32 tiles by TMA, hi/lo split in shared memory, 3 MMAs per K-block,
    split-K over a cluster with a DSMEM reduction), swapped (M <= 256) and normal orientation, ragged M / N / K, against float64.  Half of
    the rows are gradient-like (1e-7): they must not be flushed."""
    M, N, K = shape
    g = torch.Generator().manual_seed(M * 13 + N)
    x = torch.randn(M, K, generator=g)
    x[M // 2:] *= 1e-7
    w = (torch.rand(N, K, generator=g) * 2 - 1) / K ** 0.5
    b = torch.randn(N, generator=g) * 1e-3
    ref = x.double() @ w.double().t() + b.double()
    y = _linear(L, x.cuda(), w.cuda(), b.cuda(), False, 'tf32x3_tc').cpu().double()
    scale = (x.double().abs() @ w.double().abs().t() + b.double().abs())
    rel = float(((y - ref).abs() / scale).max())
    assert rel < 4e-6, (shape, rel)


@pytest.mark.parametrize('shape', [(50, 2048, 4096), (50, 1000, 9488), (360, 1024, 3072), (1000, 1024, 9488), (20, 48, 164)])
def test_tf32x3_tcgen05_input_gradient(L, shape):
    """dx[M, in] = dy[M, out] * W[out, in] through the cached transpose of W."""
    M, N, K = shape                       # N = in features, K = out features
    g = torch.Generator().manual_seed(M + N)
    dy = torch.randn(M, K, generator=g) * 1e-6
    w = (torch.rand(K, N, generator=g) * 2 - 1) / K ** 0.5
    ref = dy.double() @ w.double()
    y = torch.empty(M, N, device='cuda')
    dyd, wd = dy.cuda(), w.cuda()               # keep the device tensors alive across the asynchronous call
    L.check(L.load().capb200_linear(L.ptr(dyd), K, L.ptr(wd), N, None, L.ptr(y), N, M, N, K, 0, L.OP_MODES['tf32x3_tc_dgrad'], L.current_stream()),
            'linear dgrad')
    torch.cuda.synchronize()
    scale = dy.double().abs() @ w.double().abs()
    assert float(((y.cpu().double() - ref).abs() / scale).max()) < 4e-6


@pytest.mark.parametrize('shape', [(4096, 1024, 1000), (9488, 1024, 1000), (2048, 2048, 360), (512, 1000, 950), (96, 40, 135)])
def test_tf32x3_tcgen05_weight_gradient(L, shape):
    """dW[out, in] = dY[rows, out]^T * X[rows, in], batched over time (rows = T * N), through per-call transposes."""
    M, N, K = shape                       # M = out features, N = in features, K = rows
    g = torch.Generator().manual_seed(M + K)
    dy = torch.randn(K, M, generator=g) * 1e-6
    x = torch.randn(K, N, generator=g)
    ref = dy.double().t() @ x.double()
    y = torch.empty(M, N, device='cuda')
    dyd, xd = dy.cuda(), x.cuda()
    L.check(L.load().capb200_linear(L.ptr(dyd), M, L.ptr(xd), N, None, L.ptr(y), N, M, N, K, 0, L.OP_MODES['tf32x3_tc_wgrad'], L.current_stream()),
            'linear wgrad')
    torch.cuda.synchronize()
    scale = dy.double().abs().t() @ x.double().abs()
    assert float(((y.cpu().double() - ref).abs() / scale).max()) < 4e-6


@pytest.mark.parametrize('mode', ['simt_fp32', 'tc_f16x3'])
def test_lstm_cell(L, mode):
    g = torch.Generator().manual_seed(3)
    M, Kx, H = 37, 72, 40
    x, h, c = torch.randn(M, Kx, generator=g), torch.randn(M, H, generator=g), torch.randn(M, H, generator=g)
    cell = torch.nn.LSTMCell(Kx, H)
    with torch.no_grad():
        h_ref, c_ref = cell(x, (h, c))
    dev = [t.detach().cuda().contiguous() for t in (x, h, c, cell.weight_ih, cell.weight_hh, cell.bias_ih, cell.bias_hh)]
    ho, c_o = torch.empty(M, H, device='cuda'), torch.empty(M, H, device='cuda')
    L.check(L.load().capb200_lstm_cell(L.ptr(dev[0]), Kx, L.ptr(dev[1]), L.ptr(dev[2]), L.ptr(dev[3]), L.ptr(dev[4]), L.ptr(dev[5]), L.ptr(dev[6]),
                                       L.ptr(ho), L.ptr(c_o), M, H, L.MODES[mode], L.current_stream()), 'lstm_cell')
    torch.cuda.synchronize()
    assert float((ho.cpu() - h_ref).abs().max()) < 2e-6 and float((c_o.cpu() - c_ref).abs().max()) < 2e-6


@pytest.mark.parametrize('rpi,masked,B,A,H', [(1, False, 3, 64, 100), (5, False, 3, 64, 100), (7, True, 3, 64, 100), (10, False, 3, 64, 100),
                                               (5, False, 130, 512, 1000), (3, True, 121, 200, 300), (1, False, 150, 128, 64)])
def test_additive_attention(L, rpi, masked, B, A, H):
    """Small cases and decode-sized ones (>= 120 images, att_hid_size up to the config's 512: the score is a sum of A approximated tanh terms,
    so the bar scales with A)."""
    g = torch.Generator().manual_seed(rpi)
    R = 36
    N = B * rpi
    W = {'core.attention.h2att.weight': torch.zeros(A, H), 'core.attention.h2att.bias': torch.zeros(A),
         'core.attention.alpha_net.weight': torch.randn(1, A, generator=g), 'core.attention.alpha_net.bias': torch.randn(1, generator=g)}
    att_h = torch.randn(N, A, generator=g)
    p_att = torch.randn(B, R, A, generator=g)
    att = torch.randn(B, R, H, generator=g)
    mask = None
    if masked:
        mask = torch.ones(B, R)
        mask[0, 20:] = 0
        mask[2, 5:] = 0
        mask[B - 1, 1:] = 0
    # oracle: feed att_h through a zero h2att by adding it to p_att rows
    rep = lambda t: co.repeat_rows(t, rpi)
    dot = torch.tanh(rep(p_att) + att_h.unsqueeze(1))
    score = (dot @ W['core.attention.alpha_net.weight'].t()).squeeze(-1) + W['core.attention.alpha_net.bias']
    wgt = torch.softmax(score, 1)
    if mask is not None:
        wgt = wgt * rep(mask)
        wgt = wgt / wgt.sum(1, keepdim=True)
    ref = torch.bmm(wgt.unsqueeze(1), rep(att)).squeeze(1)
    out = torch.empty(N, H, device='cuda')
    d = [t.cuda().contiguous() if t is not None else None for t in (att_h, p_att, att, mask, W['core.attention.alpha_net.weight'], W['core.attention.alpha_net.bias'])]
    L.check(L.load().capb200_additive_attention(L.ptr(d[0]), L.ptr(d[1]), L.ptr(d[2]), L.ptr(d[3]), L.ptr(d[4]), L.ptr(d[5]), L.ptr(out), B, rpi, R, A, H,
                                                L.current_stream()), 'attention')
    torch.cuda.synchronize()
    assert float((out.cpu() - ref).abs().max()) < (5e-6 if A <= 64 else 3e-5)


@pytest.mark.parametrize('V1,twice,k,case', [(61, 0, 3, 'dense'), (9488, 1, 5, 'dense'), (9488, 0, 10, 'dense'), (1000, 1, 1, 'dense'),
                                            (9488, 1, 16, 'dense'), (9488, 1, 5, 'pitched'), (9488, 1, 16, 'owned')],
                         ids=['61-0-3', '9488-1-5', '9488-0-10', '1000-1-1', '9488-1-16', '9488-1-5-pitched', '9488-1-16-owned'])
def test_log_softmax_topk(L, V1, twice, k, case):
    """'pitched': the rows sit in a slab of pitch V1 + 4 whose other columns hold 1e30 and must be neither read nor written.
    'owned': in every row the k best all belong to one thread of the 256-thread kernel (columns congruent modulo 256)."""
    g = torch.Generator().manual_seed(V1 + k)
    rows = 17
    x = torch.randn(rows, V1, generator=g) * 4
    if case == 'owned':
        for r in range(rows):
            cols = torch.arange(r * 13 % 256, V1, 256)[torch.randperm(V1 // 256, generator=g)[:k]]
            x[r, cols] = 20.0 + 0.5 * torch.randperm(k, generator=g).float()
    ref = torch.log_softmax(x, 1)
    if twice:
        ref = torch.log_softmax(ref, 1)
    tv, ti = ref.topk(k, dim=1)
    ld = V1 + 4 if case == 'pitched' else V1
    slab = torch.full((rows, ld), 1e30, device='cuda')
    slab[:, :V1] = x.cuda()
    xd = slab[:, :V1]
    top_val = torch.empty(rows, k, device='cuda')
    top_idx = torch.empty(rows, k, dtype=torch.int32, device='cuda')
    L.check(L.load().capb200_log_softmax_topk(L.ptr(xd), ld, rows, V1, twice, k, L.ptr(top_val), L.ptr(top_idx), L.current_stream()), 'log_softmax_topk')
    torch.cuda.synchronize()
    assert float((xd.cpu() - ref).abs().max()) < 1e-5
    assert bool((slab[:, V1:] == 1e30).all())
    assert np.array_equal(top_idx.cpu().numpy(), ti.numpy().astype(np.int32))
    assert float((top_val.cpu() - tv).abs().max()) < 1e-5


def test_ciderd_reward_matches_golden(golden_dir):
    import imagecaptioning.pytorch_b200 as b200
    from oracle import ciderd_oracle as cdo
    g = np.load(os.path.join(golden_dir, 'ciderd.npz'))
    df = {tuple(int(t) for t in k if t >= 0): float(v) for k, v in zip(g['df_keys'], g['df_vals'])}
    V, B, n, T = (int(v) for v in g['meta'])
    table = b200.rewards.CiderDTable(df, float(g['ref_len']))
    gts = [g['gts'][i] for i in range(B)]
    scores, reward = b200.rewards.cider_scores_and_reward(torch.from_numpy(g['greedy']).cuda(), gts, torch.from_numpy(g['sampled']).cuda(), table)
    torch.cuda.synchronize()
    assert np.abs(scores.cpu().numpy()[:B * n] - g['sample_scores']).max() < 1e-9
    assert np.abs(reward.cpu().numpy() - g['reward']).max() < LOGP_TOL
    # ragged references + random hypotheses against the oracle
    rng = np.random.RandomState(5)
    gts2 = [cdo.make_refs(1, V, n_refs=int(rng.randint(1, 6)), seed=int(s))[0] for s in rng.randint(0, 1000, size=7)]
    samp = np.minimum(rng.zipf(1.3, size=(7 * 3, 20)), V).astype(np.int64)
    samp[rng.rand(*samp.shape) < 0.08] = 0
    grd = np.minimum(rng.zipf(1.3, size=(7, 20)), V).astype(np.int64)
    ref_reward, ref_scores = cdo.self_critical_reward(grd, gts2, samp, df, float(g['ref_len']))
    scores, reward = b200.rewards.cider_scores_and_reward(torch.from_numpy(grd).cuda(), gts2, torch.from_numpy(samp).cuda(), table)
    assert np.abs(scores.cpu().numpy() - ref_scores).max() < 1e-9
    assert np.abs(reward.cpu().numpy() - ref_reward).max() < LOGP_TOL


def test_reward_criterion_matches_golden(golden_dir):
    import imagecaptioning.pytorch_b200 as b200
    g = np.load(os.path.join(golden_dir, 'reward_criterion.npz'))
    lp, seq, reward = (torch.from_numpy(g[k]).cuda() for k in ('lp', 'seq', 'reward'))
    crit = b200.RewardCriterion()
    loss = crit(lp, seq, reward)
    assert abs(float(loss) - float(g['loss'])) < 1e-6
    assert np.abs(crit(lp, seq, reward, reduction='none').cpu().numpy() - g['loss_none']).max() < 1e-6
    grad = crit.backward_logprobs(seq, reward, lp.shape[2])
    assert np.abs(grad.cpu().numpy() - g['grad']).max() < 1e-7


@pytest.mark.parametrize('clip,wd', [(None, 0.0), (0.05, 0.0), (0.05, 0.01)])
def test_fused_adam_matches_torch_adam(clip, wd):
    """capb200_adam_step (clamp + Adam in one launch; tools/train.py:193-196) against utils.clip_gradient's clamp + torch.optim.Adam over four
    steps: parameters, both moment buffers and the clamped gradients; odd sizes and a misaligned view exercise the scalar tails; the state
    dict written by one loads into the other."""
    import imagecaptioning.pytorch_b200 as b200
    g = torch.Generator(device='cuda').manual_seed(3)
    shapes = [(1000, 37), (4097,), (3, 5, 7), (1,), (8192 * 2 + 5,)]
    mine = [torch.nn.Parameter(torch.randn(s, generator=g, device='cuda')) for s in shapes]
    mine.append(torch.nn.Parameter(torch.randn(1001, generator=g, device='cuda')[1:]))      # a view that is only 4-byte aligned
    ref = [torch.nn.Parameter(t.detach().clone()) for t in mine]
    o_mine = b200.optim.FusedAdam(mine, lr=3e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=wd, clip_value=clip)
    o_ref = torch.optim.Adam(ref, lr=3e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=wd)
    for it in range(4):
        for a, b in zip(mine, ref):
            gr = torch.randn(a.shape, generator=g, device='cuda') * (0.1 if it % 2 else 1.0)
            a.grad = gr.clone()
            b.grad = gr.clone()
        if clip:
            for b in ref:
                b.grad.data.clamp_(-clip, clip)             # captioning/utils/misc.py:156-160
        o_mine.step()
        o_ref.step()
        for a, b in zip(mine, ref):
            scale = float(b.abs().max()) + 1e-6
            assert float((a - b).abs().max()) <= 2e-6 * scale
            assert torch.equal(a.grad, b.grad)
            sa, sb = o_mine.state[a], o_ref.state[b]
            assert float((sa['exp_avg'] - sb['exp_avg']).abs().max()) <= 1e-6 * (float(sb['exp_avg'].abs().max()) + 1e-12)
            assert float((sa['exp_avg_sq'] - sb['exp_avg_sq']).abs().max()) <= 1e-6 * (float(sb['exp_avg_sq'].abs().max()) + 1e-12)
            assert float(sa['step']) == float(sb['step']) == it + 1
    assert o_mine.launches == 4
    o_ref.load_state_dict(o_mine.state_dict())              # same layout: optimizer.pth is interchangeable (tools/train.py:74-77)
    o_mine.load_state_dict(o_ref.state_dict())
