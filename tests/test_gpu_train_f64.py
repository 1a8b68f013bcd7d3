"""The fused training steps of UpDown, Att2in2, NewFC, AoANet and the Transformer at the widths they train at, PPO's included, against
float64 autograd through the oracle.

UpDown runs at bench.py's CFG (V 9487, E = H = 1000, A 512, F 2048), Att2in2 at the a2i2 recipe width (E = H = A = 512), AoANet at
configs/aoa.yml's (E = H = 1024, 8 heads, 6 refiner layers) and the Transformer at bench.py's transformer_scst (6 + 6 layers, d_model 512,
d_ff 2048, 8 heads), all with 36 regions and 20 steps.  In both modes the vocabulary-row kernels
loop 37 times per row, the attention backward runs 16 column blocks per image and the autograd VJP takes its 4-wide form.  The training
GEMMs differ by mode: tc_f16x3 runs them on gemm_tf32.cu's wgmma 3xTF32 kernel, whose tile follows the row count (50 rows per step: tile
width 64, swapped; 1000 rows batched over time: the normal orientation, cluster split-K over K = 9488 for the logit layer); simt_fp32 runs
gemm_generic.cu's CUDA-core kernels with their one tile shape.

Every case compares loss, picked log-probs, reward and every parameter gradient with the same step run through the oracle in float64.  The
bar calibrates itself: the step also runs through the oracle in float32, and each tensor's error may be at most
    max(4 x the fp32 oracle's error, 2e-6 x max|f64|) + 1e-7 x the step's largest gradient entry,
(the 2e-6 grows as sqrt(N * T / 1000) past 1000 reduced (step, row) pairs),
in max-abs and in Frobenius norm.  Samples and baseline captions are replayed (forced_tokens / forced_baseline), so no near-tie in sampling
can change what is compared.

Kinks: a ReLU input or a maxout pair within rounding of the switch point can land on either side in fp32.  The float64 pass lists those
units (margin KINK_MARGIN x the layer's RMS, several times the fp32 error of these dot products):
* ReLU (att_embed, fc_embed): the gradient through unit j only reaches row j of the layer's weight and entry j of its bias, so those
  entries are left out;
* Att2in2's maxout: the routed gradient runs back through the recurrence into every core tensor, so leaving entries out would drop whole
  tensors.  Instead the gradient change of re-routing each ambiguous unit is computed in float64 (one caption row rerun), and for each unit
  the side that fits the engine better is taken.  Each change is hundreds of times the bar, so the choice is never close.
The fp32 oracle follows float64's decisions at every kink, so its distance from float64 is arithmetic only.

The Transformer's feed-forward ReLUs feed the residual stream, so a flipped unit moves the gradient of every tensor upstream of it, and
they are too many to re-route one by one (about 250 units per encoder layer and 650 per decoder layer lie within 5e-4 x RMS of zero).
Instead each case moves its model off the kinks before anything runs (helpers.clear_relu_kinks): in layer order, every att_embed or w_1
unit with a float64 input within TFM_MARGIN x the layer's RMS of zero gets its bias shifted by the smallest +-k x margin x RMS that clears
all its rows, and the engine and all oracles then use those fp32 weights.  Every float64 ReLU input is asserted to clear the margin, and
5x the calibrating oracle's largest error there to stay below it, so no tensor is left out.  Measured on an H100 at 50 rows per step: the
fp32 oracle's error there is 3.7-4.5e-6 x RMS and the 3xTF32 emulation's 0.95-1.12e-4 x RMS (5x = 0.59-0.70 of the 8e-4 margin); 100 att_embed
units and 200-970 per feed-forward layer move, by at most 1.4e-2 x RMS.  At 160 rows per step (3360 decoder rows) 1000-1750 units per
layer move, by at most 9.8e-2 x RMS: the rows crowd each unit's band, so the clearing shift is larger, but every unit clears within 200
margins.  The engine fuses the q | k | v and the memory k | v projections into one GEMM each; an output column of a GEMM depends only on
its weight row and the K loop, so the emulation's separate Linears bound them column by column (split-K follows the tile count, and the
emulation's single accumulator is the larger truncation count either way).

Calibration per mode: simt_fp32 is held to the fp32 oracle.  tc_f16x3 is held to the same oracle with every Linear's forward and input
gradient computed as gemm_tf32 does (_mm_tf32x3): hi / lo tf32 split, three wgmmas per k8 step into one fp32 accumulator, and the
accumulator truncated (rounded toward zero) by every instruction, the budget test_gpu_ops.py already gives this kernel.  Over K = 3000
that is 1125 truncations, biased toward zero, so the mode's log-probs and gradients sit 10-40x further from float64 than fp32's; the
emulation reproduces that (its picked log-probs sit 1-3x the engine's distance from float64) and the bar is 4x its error, as for fp32.
It over-counts the forward's truncations (the kernel's cluster split-K gives each CTA a slice of K) and leaves the weight gradients, which
the engine batches over time, in fp32, so it is no tighter bound than that: at 320 rows the engine's logit.weight gradient reaches 1.25x
the emulation's error.  That slack limits what tc_f16x3 can see in the weight gradients: with one of the three products (hi(dY) x lo(X))
dropped from every Transformer weight gradient, the worst err/bar rose from 0.11 to 0.85 (src_attn.linears.1.weight) and the case still
passed.  simt_fp32, held to the fp32 oracle, is the mode that catches errors of 1e-4 of a tensor.

Att2in2 runs in simt_fp32 only.  In tc_f16x3 the engine's own error in the maxout inputs is of the order of the kink margin, and the
gradient change of re-routing a unit is no longer decisive against the mode's error, so the maxout decisions cannot be read off.

NewFC runs at the fc_rl / fc_nsc recipe width (E = H = 512, F_fc 2048, logit_scale 12 as its recipe-size golden), in both modes: its
maxout decisions are decisive in tc_f16x3 too (5-6 ambiguous units per case, none re-routed).  Its simt_fp32 logit.weight gradient is what
made gemm_generic_kernel sum each K-tile apart before adding it to the running total: with one accumulator over the 1000 (step, row) pairs
it sat 3e-6 of the tensor's largest entry from float64 in the greedy case without dropout (1.38x the bar; torch's blocked fp32 sum: 4e-7).

PPO (kind 'ppo', ppo_step) is compared as the other kinds, with the old policy's teacher-forced pass over [0, samples[:, :-1]] in eval mode
taken as a constant and the backward through the new policy only.  Each case's cliprange is the first of CLIPRANGES whose edges no float64
ratio comes within 1e-4 of (at an edge the picked word's gradient jumps between -adv x ratio and 0), both branches are asserted to run, and
the engine's clipfrac must equal float64's count over the mask sum as an fp32 value.  simt_fp32 is calibrated by the fp32 oracle for both
policies; tc_f16x3 by the 3xTF32 emulation for the new policy and by the old engine's own eval-mode teacher-forced log-probs (the path the
step's old pass takes), which are held to float64 within LOGP_TOL at every position the mask keeps: the bar therefore does not cover
errors of the old pass below that tolerance.  From the engine's own log-probs and scores, loss, pg_loss, kl_loss and clipfrac are also
recomputed in float64 and held to the summation bound, which checks ppo_mask / row / reduce_kernel apart from the model's arithmetic.

The loss is a sum over every caption position, reduced in another order than torch's; its floor is the pairwise-summation bound
2^-24 x log2(terms) x sum of |terms| rather than a fixed 1e-6.
"""
import contextlib
import time

import numpy as np
import pytest
import torch

import att2in2_oracle as ao
import newfc_oracle as no
from helpers import (LOGP_TOL, aoa_masks, att2in2_masks, check_grads_f64, clear_relu_kinks, co, dropout_masks, family_opt, ffn_relu_inputs,
                     tfm_masks)
from ppo_oracle import old_policy_input, ppo_loss, token_mask

pytestmark = pytest.mark.gpu

R, T, SPI, HEADS = 36, 20, 5, 8
CFGS = {'updown': dict(V=9487, E=1000, H=1000, A=512, F_fc=2048, F_att=2048, T=T),      # bench.py CFG
        'att2in2': dict(V=9487, E=512, H=512, A=512, F_fc=2048, F_att=2048, T=T),       # a2i2 recipe
        'newfc': dict(V=9487, E=512, H=512, A=512, F_fc=2048, F_att=2048, T=T),         # fc_rl / fc_nsc recipe (golden/newfc_cfg1.npz)
        'aoa': dict(V=9487, E=1024, H=1024, A=0, F_fc=2048, F_att=2048, T=T),           # configs/aoa.yml
        'transformer': dict(V=9487, E=512, H=2048, A=6, F_fc=2048, F_att=2048, T=T)}    # bench.py transformer_scst: d_model, d_ff, layers
# bench.py's synthetic models; NewFC, which bench.py does not train, takes the 12.0 of its recipe-size golden (golden/newfc_scst_full.npz)
LOGIT_SCALE = {'updown': 12.0, 'att2in2': 12.0, 'newfc': 12.0, 'aoa': 6.0, 'transformer': 3.0}
RATES = {'updown': 0.5, 'att2in2': 0.5, 'newfc': 0.5, 'aoa': (0.5, 0.1, 0.3, 0.1),       # drop_prob_lm (+ AoANet: attention, AoA, sublayer)
         'transformer': (0.5, 0.1)}                                                       # drop_prob_lm, dropout (transformer.yml, opts)
MAXOUT = ('att2in2', 'newfc')   # the families whose core is co.maxout_lstm
SAMPLED = ('greedy', 'leave_one_out', 'ppo')
# PPO: the cliprange of a case is the first of these whose edges 1 -+ eps no float64 policy ratio comes within CLIP_MARGIN of, so that the
# clipped surrogate takes the same branch in every implementation; KL_COEF is the reference's default, KL_COEF_FULL lets the full-row KL
# gradient stand out of the policy-gradient term
CLIPRANGES, CLIP_MARGIN = (0.2, 0.15, 0.25, 0.1, 0.3), 1e-4
KL_COEF, KL_COEF_FULL = 0.02, 1.0
PPO_KEEP = 30                   # drop_worst: the loss of the 30 best of 50 rows
# the old policy's weights are the new ones plus this much noise (relative to each tensor's spread): a quarter to a half of the ratios of
# each perturbed case leave the clip range (_ppo_reference asserts some do and some do not)
PERTURB = {'updown': 0.2, 'att2in2': 0.1, 'newfc': 0.05, 'aoa': 0.25, 'transformer': 0.05}
KINK_MARGIN = 2e-5              # ReLU inputs and maxout a - b: x the layer's RMS, at least 5x the fp32 oracle's own error there (asserted)
TFM_MARGIN = 8e-4               # the Transformer's ReLU inputs are moved this far (x the layer's RMS) from zero; 5x the calibrating oracle's
                                # error there must stay below it (asserted; the 3xTF32 emulation's is the larger, 1e-4)
SEED = 4242
COLLIDE = 7                     # the word that fills whole caption rows: embed_scatter's atomics all land on one row of d_emb

_MODELS, _WEIGHTS = {}, {}
_CASES = {}                     # each case's float64 / fp32 references, held until every mode has been compared with them


def _tf32(x, nearest):
    """x (fp32) cut to tf32's 10 explicit mantissa bits: to nearest with ties away from zero (cvt.rna.tf32), or toward zero (what the
    tensor core keeps of the fp32 lo operand)."""
    i = x.contiguous().view(torch.int32)
    return ((i + 0x1000 if nearest else i) & ~0x1FFF).view(torch.float32)


def _mm_tf32x3(a, b):
    """a [M, K] @ b [K, N] as gemm_tf32.cu computes it, on the GPU: hi = rna(x), lo = x - hi as the tensor core keeps it, and per k8 step
    three wgmmas (hi.lo, lo.hi, hi.hi) into one fp32 accumulator that every instruction truncates (rounds toward zero).  The products of a
    k8 step are summed exactly (float64); each truncation is taken at the exact running sum, which leaves out only the second-order effect
    of earlier truncations on later ones.  The whole K runs through one accumulator (the kernel's cluster split-K gives each CTA a slice
    and sums the slices rounded to nearest, so this is the larger of the two truncation counts)."""
    dev = torch.device('cuda')
    a, b = a.detach().to(dev, torch.float32), b.detach().to(dev, torch.float32)
    M, K = a.shape
    N = b.shape[1]
    Kp = -(-K // 8) * 8
    a, b = torch.nn.functional.pad(a, (0, Kp - K)), torch.nn.functional.pad(b.t(), (0, Kp - K))      # [M, Kp], [N, Kp]
    ah, bh = _tf32(a, True), _tf32(b, True)
    al, bl = _tf32(a - ah, False), _tf32(b - bh, False)
    J = Kp // 8
    out = torch.empty(M, N, dtype=torch.float64, device=dev)
    rows = max(1, int(2e8 // (N * J * 3)))
    for m0 in range(0, M, rows):
        sl = slice(m0, m0 + rows)

        def step(x, y):
            return torch.einsum('mjb,njb->mnj', x[sl].double().view(-1, J, 8), y.double().view(N, J, 8))
        seq = torch.stack([step(ah, bl), step(al, bh), step(ah, bh)], -1).flatten(2)          # [m, N, 3J], in issue order
        run = seq.cumsum(-1)
        f = run.float()
        f = torch.where(f.double().abs() > run.abs(), torch.nextafter(f, torch.zeros_like(f)), f)     # round toward zero
        out[sl] = run[..., -1] + (f.double() - run).sum(-1)
        del seq, run, f
    return out.float().cpu()


class _Tf32x3Linear(torch.autograd.Function):
    """x @ w.T with the forward and the input gradient as gemm_tf32 computes them; the weight gradient in plain fp32."""
    @staticmethod
    def forward(ctx, x, w):
        ctx.save_for_backward(x, w)
        return _mm_tf32x3(x.reshape(-1, x.shape[-1]), w.t()).reshape(*x.shape[:-1], w.shape[0])

    @staticmethod
    def backward(ctx, gy):
        x, w = ctx.saved_tensors
        g2 = gy.reshape(-1, gy.shape[-1])
        return _mm_tf32x3(g2, w).reshape(x.shape), g2.t() @ x.reshape(-1, x.shape[-1])


def _tf32x3_linear(x, w, b=None):
    y = _Tf32x3Linear.apply(x, w)
    return y if b is None else y + b


@contextlib.contextmanager
def _linear(fn):
    orig = co.linear
    co.linear = fn
    try:
        yield
    finally:
        co.linear = orig


@contextlib.contextmanager
def _routed_maxout(record, route=None, flip=None):
    """co.maxout_lstm with its routing exposed: each call appends a - b of the two maxout halves to ``record``; ``route`` (one bool [N, H]
    per step) fixes which half takes the gradient, and ``flip`` {step: bool [N, H]} re-routes single units.  The forward value is always
    max(a, b)."""
    orig, step = co.maxout_lstm, [0]

    def maxout_lstm(W, x, state):
        h, c = state
        hs = h.shape[2]
        s = co.linear(x, W['_core.i2h.weight'], W['_core.i2h.bias']) + co.linear(h[-1], W['_core.h2h.weight'], W['_core.h2h.bias'])
        sig = torch.sigmoid(s[:, :3 * hs])
        a, b = s[:, 3 * hs:4 * hs], s[:, 4 * hs:5 * hs]
        record.append((a - b).detach())
        t = step[0]
        step[0] += 1
        sel = (a > b) if route is None else route[t]
        if flip is not None and t in flip:
            sel = sel ^ flip[t]
        routed = torch.where(sel, a, b)
        g = routed + (torch.maximum(a, b) - routed).detach()
        c_new = sig[:, hs:2 * hs] * c[-1] + sig[:, :hs] * g
        h_new = sig[:, 2 * hs:] * torch.tanh(c_new)
        return h_new, (h_new.unsqueeze(0), c_new.unsqueeze(0))
    co.maxout_lstm = maxout_lstm
    try:
        yield
    finally:
        co.maxout_lstm = orig


def _weights(family):
    if family not in _WEIGHTS:
        c = CFGS[family]
        _WEIGHTS[family] = co.make_weights(family, c['V'], c['E'], c['H'], c['A'], c['F_fc'], c['F_att'], seed=1, logit_scale=LOGIT_SCALE[family])
    return _WEIGHTS[family]


def _model(family, mode, autograd=False, old=False):
    """The engine model of (family, mode); ``old``: a second one, PPO's frozen old policy."""
    import imagecaptioning.pytorch_b200 as b200
    key = (family, mode, autograd, old)
    if key not in _MODELS:
        c = CFGS[family]
        opt = family_opt(family, c['V'], c['E'], c['H'], c['A'], c['F_fc'], c['F_att'], T, heads=HEADS)
        opt.b200_autograd = int(autograd)
        m = b200.setup(opt, numeric_mode=mode)
        m.load_state_dict(_weights(family), strict=True)
        _MODELS[key] = m.cuda()
    return _MODELS[key]


def _region_masks(B):
    """Prefix masks: image 0 keeps all 36 regions, the others 3 to 35, several of them fewer than 10."""
    m = torch.zeros(B, R)
    for i in range(B):
        m[i, :R if i == 0 else [7, 20, 3, 35, 9, 28, 5, 14, 31][(i - 1) % 9]] = 1
    return m


def _samples(gts, B, V, seed):
    """Forced samples [B * 5, T] built from each image's references (so CIDEr-D rewards differ from row to row) with edges: row 0 is EOS
    at t = 0; image 1's five samples are identical; every even row of the even images runs all T steps without EOS; image 3's rows are
    COLLIDE at every step but one, image 4's at every other step."""
    rng = np.random.RandomState(seed)
    tok = np.zeros((B * SPI, T), np.int64)
    for i in range(B * SPI):
        b, j = divmod(i, SPI)
        ref = [w for w in gts[b][j % len(gts[b])] if w > 0]
        words = [w if rng.rand() > 0.3 else int(rng.randint(1, V + 1)) for w in ref]
        full = b % 2 == 0 and j % 2 == 0
        ln = T if full else int(rng.randint(1, T))
        while len(words) < ln:
            words.append(int(min(rng.zipf(1.3), V)))
        tok[i, :ln] = words[:ln]
    tok[0] = 0
    if B > 1:
        tok[SPI:2 * SPI] = tok[SPI]
    if B > 4:
        for j in range(SPI):
            r3, r4 = 3 * SPI + j, 4 * SPI + j
            tok[r3] = COLLIDE
            tok[r3, j] = tok[r4, j] if tok[r4, j] else 1
            tok[r4, ::2] = COLLIDE
            tok[r4, 1::2] = np.where(tok[r4, 1::2] > 0, tok[r4, 1::2], 2)
    return torch.from_numpy(tok)


def _labels(gts, B, V, seed):
    """XE labels [B, 5, T + 2] of mixed lengths 1 .. T (BOS at 0, EOS after the last word) built from the references, image 3's rows
    filled with COLLIDE, and their masks."""
    tok = _samples(gts, B, V, seed)
    tok[0, :3] = torch.tensor([5, 6, 7])          # the sampler's EOS-first row has no XE counterpart: a 3-word caption instead
    labels = torch.zeros(B * SPI, T + 2, dtype=torch.long)
    masks = torch.zeros(B * SPI, T + 2)
    for i in range(B * SPI):
        ln = int((tok[i] > 0).cumprod(0).sum())
        labels[i, 1:1 + ln] = tok[i, :ln]
        masks[i, :ln + 2] = 1
    return labels.view(B, SPI, -1), masks.view(B, SPI, -1)


class Case:
    def __init__(self, family, kind, dropout, B, smoothing=0.0, regions=False, ppo=None):
        """``ppo`` (kind 'ppo'): (perturbation of the old policy's weights, kl_coef, keep_rows)."""
        from oracle import ciderd_oracle as cdo
        self.family, self.kind, self.dropout, self.B, self.smoothing = family, kind, dropout, B, smoothing
        c = CFGS[family]
        self.c, self.N = c, B * SPI
        self.fc, self.att = co.make_inputs(B, R, c['F_fc'], c['F_att'], seed=17)
        if family == 'newfc':                   # NewFC reads no region features: what the reference loader hands it
            self.att = self.fc.new_zeros(B, 0, 0)
        self.regions = _region_masks(B) if regions else None
        self.Rc = R if self.regions is None else int(self.regions.sum(1).max())
        self.gts = cdo.make_refs(B, c['V'], seed=5)
        self.df, self.ref_len = cdo.build_document_frequency(cdo.make_refs(1000, c['V'], seed=4))
        self.steps = T + 1 if kind in ('xe', 'autograd') else T
        if kind in SAMPLED:
            self.tok = _samples(self.gts, B, c['V'], seed=23)
            self.base = torch.stack([torch.from_numpy(np.pad(self.gts[b][1][:9], (0, T - 9))) for b in range(B)])
            if kind == 'greedy':
                reward, _ = cdo.self_critical_reward(self.base.numpy(), self.gts, self.tok.numpy(), self.df, self.ref_len)
            else:
                sc = cdo.get_scores(self.gts, self.tok.numpy(), self.df, self.ref_len).reshape(B, SPI)
                adv = (sc - (sc.sum(1, keepdims=True) - sc) / (SPI - 1)).reshape(-1, 1)
                # PPO's reward is the scores themselves (the step returns them), its advantage their leave-one-out form
                reward = sc.reshape(-1) if kind == 'ppo' else np.repeat(adv, T, 1)
                self.adv = torch.from_numpy(adv.reshape(-1)).double()
            self.reward = torch.from_numpy(np.ascontiguousarray(reward)).double()
            self.mask = torch.cat([torch.ones(self.N, 1), (self.tok[:, :-1] > 0).double()], 1)
            assert torch.equal(self.mask, token_mask(self.tok))
        else:
            self.labels, self.lmasks = _labels(self.gts, B, c['V'], seed=29)
            self.tl, self.tm = self.labels[..., 1:].reshape(self.N, -1), self.lmasks[..., 1:].reshape(self.N, -1)
            if kind == 'autograd':
                self.G = torch.randn(self.N, T + 1, c['V'] + 1, generator=torch.Generator().manual_seed(31))
        if kind == 'ppo':
            self.perturb, self.kl_coef, self.keep_rows = ppo
            self.eps = None                     # chosen by the float64 pass (_cliprange)
            self._lo = {}
        self.drop = None
        self.W = _weights(family)             # the Transformer's are moved off its ReLU kinks for each case (reference())

    # ---- the step through the oracle ----------------------------------------------------------------------------------------------------
    def _family(self, W):
        if self.family == 'att2in2':
            return ao.Att2in2Family(W, T)
        if self.family == 'newfc':
            return no.NewFCFamily(W, T)
        return co.Family(self.family, W, T, heads=HEADS)

    def _old_weights(self):
        """PPO's old policy: this case's weights, each tensor plus perturb x its spread of seeded noise."""
        if not self.perturb:
            return dict(self.W)
        g = torch.Generator().manual_seed(SEED)
        return {k: v if k.endswith('.pe') else v + self.perturb * (float(v.std()) if v.numel() > 1 else 1.0) * torch.randn(v.shape, generator=g)
                for k, v in self.W.items()}

    def old_lp(self, dt):
        """PPO's old policy in dtype dt: eval mode (no dropout), teacher-forced over [0, samples[:, :-1]]; [N, T, V + 1], zero past the
        column where every row has ended."""
        if dt not in self._lo:
            fam = self._family({k: v.to(dt) for k, v in self.W_old.items()})
            with torch.no_grad():
                self._lo[dt] = co.forward_teacher(fam, self.fc.to(dt), self.att.to(dt), old_policy_input(self.tok).view(self.B, SPI, -1), self.regions)
        return self._lo[dt]

    def _cliprange(self, lp, lo):
        """The first of CLIPRANGES whose edges no float64 ratio at a position the PPO mask keeps comes within CLIP_MARGIN of."""
        ratio = self._ratios(lp, lo)
        for eps in CLIPRANGES:
            if float(torch.minimum((ratio - (1 - eps)).abs(), (ratio - (1 + eps)).abs()).min()) > CLIP_MARGIN:
                return eps
        raise AssertionError('every cliprange has a ratio on its edge')

    def _ratios(self, lp, lo):
        idx = self.tok.unsqueeze(2)
        return torch.exp(lp.gather(2, idx) - lo.gather(2, idx)).squeeze(2)[self.mask > 0]

    def _inputs(self, rows, dt):
        """(fc, att, regions, drop, words) of all rows (rows None) or of one caption row."""
        fc, att, reg, drop = self.fc, self.att, self.regions, self.drop
        words = self.tok if self.kind in SAMPLED else self.labels[..., :-1].reshape(self.N, -1)
        if rows is not None:
            # row n of image b, and a companion row of COLLIDE words that runs every step (a teacher-forced pass stops at the first
            # column where every row is pad, and the full batch runs on past row n's end); only row n enters the objective
            n = rows
            b = n // SPI
            fc, att = fc[b:b + 1], att[b:b + 1]
            words = torch.cat([words[n:n + 1], torch.full_like(words[n:n + 1], COLLIDE)])
            rb = R if reg is None else int(reg[b].sum())
            if reg is not None:
                reg = reg[b:b + 1]
            if drop is not None:        # Att2in2's att, xt and out sites; NewFC's out
                drop = {k: v[b:b + 1, :rb] if k == 'att' else v[:, [n, n]] for k, v in drop.items()}
        if drop is not None:
            drop = {k: v.to(dt) for k, v in drop.items()}
        return fc.to(dt), att.to(dt), reg, drop, words

    def _objective(self, lp, rows, dt, lo=None):
        """The step's loss (all rows), or the share of it that one caption row contributes (same normaliser).  ``lo``: PPO's old-policy
        log-probs of all rows."""
        sl = slice(None) if rows is None else slice(rows, rows + 1)
        if self.kind == 'ppo':
            if rows is None:
                if self.eps is None:
                    self.eps = self._cliprange(lp.detach(), lo)
                out = ppo_loss(lp, lo, self.tok, self.reward.to(dt), SPI, self.eps, self.kl_coef, 'none' if self.keep_rows else 'mean')
                return out['loss'].sort().values[:self.keep_rows].mean() if self.keep_rows else out['loss']
            row = ppo_loss(lp, lo[sl], self.tok[sl], None, 1, self.eps, self.kl_coef, 'none', adv=self.adv[sl])['loss'][0]
            if self.keep_rows:
                return row * float(self.kept[rows]) / self.keep_rows
            return row * self.mask[sl].sum().to(dt) / self.mask.sum()
        if self.kind in ('greedy', 'leave_one_out'):
            reward = self.reward.to(dt)[sl]
            if rows is None:
                return co.reward_criterion(lp, self.tok, reward)
            tok, mask = self.tok[sl], self.mask.to(dt)[sl]
            return -(lp.gather(2, tok.unsqueeze(2)).squeeze(2) * reward * mask).sum() / self.mask.sum()
        if self.kind == 'autograd':
            return (lp * self.G.to(dt)[sl]).sum()
        tl, tm = self.tl[sl], self.tm[sl]
        if self.smoothing:
            crit = lambda *a, **k: co.label_smoothing_loss(*a, self.smoothing, **k)       # noqa: E731
        else:
            crit = co.language_model_criterion
        if rows is None:
            return crit(lp, tl, tm)
        return (crit(lp, tl, tm, reduction='none') * tm.sum(1).to(dt)).sum() / self.tm.sum()

    def _forward(self, W, dt, rows=None):
        """The step's log-probs through the oracle with weights W.  The Transformer's is always one causal teacher-forced pass: XE masks
        pad keys; the sampled steps feed [0, samples[:, :-1]] under the causal mask alone (what the sampler's cached K/V sees) and zero
        the rows of finished samples, as the sampler stores them."""
        fam = self._family(W)
        fc, att, reg, fam.drop, words = self._inputs(rows, dt)
        sampled = self.kind in SAMPLED
        if self.family == 'transformer' and sampled:
            lp = co.forward_teacher(fam, fc, att, torch.cat([torch.zeros_like(words[:, :1]), words[:, :-1]], 1), reg, pad_keys_masked=False)
            return lp * torch.cat([torch.ones_like(words[:, :1]), (words[:, :-1] > 0).long()], 1).unsqueeze(2).to(dt)
        if sampled:
            return co.sample(fam, fc, att, reg, sample_method='sample', sample_n=2 if rows is not None else SPI, forced_tokens=words)[1]
        return co.forward_teacher(fam, fc, att, words.view(fc.shape[0], -1, words.shape[1]), reg)

    def oracle(self, dt, rows=None, route=None, flip=None, record=None, tf32x3=False, lo=None):
        """(loss, log-probs, gradients) of the step in dtype dt.  ``record`` collects the maxout a - b of Att2in2 and NewFC, or the
        Transformer's ReLU inputs (att_embed's, then each feed-forward layer's).  PPO's old policy is ``lo``, by default the oracle's own
        pass in dtype dt, taken outside the hooks (no gradient flows through it)."""
        W = {k: v.detach().to(dt, copy=True).requires_grad_(not k.endswith('.pe')) for k, v in self.W.items()}       # pe: a buffer
        if self.kind == 'ppo' and lo is None:
            lo = self.old_lp(dt)
        record = [] if record is None else record
        hooks = contextlib.nullcontext()
        if self.family in MAXOUT:
            hooks = _routed_maxout(record, route, flip)
        elif self.family == 'transformer':
            hooks = ffn_relu_inputs(lambda pre, Wd, a: record.append(a.detach().reshape(-1, a.shape[-1])) or a)
        with hooks, (_linear(_tf32x3_linear) if tf32x3 else contextlib.nullcontext()):
            if self.family == 'transformer':
                record.append(co.linear(self.att.to(dt).reshape(-1, self.att.shape[-1]), W['att_embed.0.weight'], W['att_embed.0.bias']).detach())
            lp = self._forward(W, dt, rows)
        if rows is not None:
            lp = lp[:1]
        loss = self._objective(lp, rows, dt, lo)
        loss.backward()
        return float(loss), lp.detach(), {k: v.grad for k, v in W.items() if v.requires_grad}

    def picked(self, lp):
        if self.kind in SAMPLED:
            return lp.gather(2, self.tok.unsqueeze(2)).squeeze(2)
        if self.kind == 'autograd':
            return lp
        return lp.gather(2, self.tl[:, :lp.shape[1]].unsqueeze(2)).squeeze(2)

    def relu_kinks(self):
        """{parameter name: bool mask of the entries kept}: rows j of a ReLU layer's weight (and entry j of its bias) whose input lies within
        KINK_MARGIN x RMS of zero for some valid region (or image), in float64.  The fp32 pre-activations must sit well inside the margin."""
        if self.family in ('transformer', 'newfc'):  # the Transformer's ReLUs are cleared by construction (reference()); NewFC has none
            self.kink_rows = {}
            return {}, 0
        W = _weights(self.family)
        layers = [('att_embed.0', self.att)] + ([('fc_embed.0', self.fc.unsqueeze(1))] if self.family == 'updown' else [])
        keep, left_out, self.kink_rows = {}, 0, {}
        for name, x in layers:
            pre = co.linear(x.double(), W[name + '.weight'].double(), W[name + '.bias'].double())
            valid = torch.ones(pre.shape[:2], dtype=torch.bool)
            if self.regions is not None and name == 'att_embed.0':
                valid = self.regions.bool()
            rms = float(pre[valid].pow(2).mean().sqrt())
            pre32 = co.linear(x, W[name + '.weight'], W[name + '.bias'])
            assert 5 * float((pre32.double() - pre).abs().max()) < KINK_MARGIN * rms
            amb = ((pre.abs() < KINK_MARGIN * rms) & valid.unsqueeze(-1)).any(1).any(0)          # [H]
            keep[name + '.weight'] = ~amb.unsqueeze(1).expand_as(W[name + '.weight'])
            keep[name + '.bias'] = ~amb
            left_out += int(amb.sum()) * (W[name + '.weight'].shape[1] + 1)
            self.kink_rows[name] = int(amb.sum())
        return keep, left_out

    def reference(self):
        t0 = time.time()
        if self.family == 'transformer':
            self.W, self.shifted, self.largest_shift = clear_relu_kinks(_weights(self.family), self.att, lambda W: self._forward(W, torch.float64),
                                                                        TFM_MARGIN)
        if self.kind == 'ppo':
            self.W_old = self._old_weights()
        rec64, rec32 = [], []
        loss64, lp64, g64 = self.oracle(torch.float64, record=rec64)
        route = [d > 0 for d in rec64] if rec64 and self.family in MAXOUT else None
        if self.kind == 'ppo':
            self._ppo_reference(lp64)
        loss32, lp32, g32 = self.oracle(torch.float32, route=route, record=rec32)
        self.ref = dict(loss64=loss64, loss32=loss32, picked64=self.picked(lp64), picked32=self.picked(lp32).double(), g64=g64, g32=g32)
        self.ref['l1'] = self._loss_l1(lp64)
        self.keep, self.left_out = self.relu_kinks()
        self.maxout = []
        if self.family == 'transformer':
            self.relu64 = rec64
            rms = [float(a.pow(2).mean().sqrt()) for a in rec64]
            clear = min(float(a.abs().min()) / r for a, r in zip(rec64, rms))
            assert clear >= TFM_MARGIN, clear                  # every float64 ReLU input lies at least the margin from its kink
            self.relu_err = {'fp32 oracle': self._relu_err(rec32)}
        elif rec64:
            d = torch.stack(rec64)                                   # [steps, N, H]
            rms = float(d.pow(2).mean().sqrt())
            err32 = float((torch.stack(rec32).double() - d).abs().max())
            assert 5 * err32 < KINK_MARGIN * rms, (err32, rms)
            self.maxout = [tuple(int(v) for v in u) for u in (d.abs() < KINK_MARGIN * rms).nonzero()]
            self.route = route
        self.ref_seconds = time.time() - t0

    def _ppo_reference(self, lp64):
        """PPO's float64 decisions: the clip count over the mask sum, and for drop_worst the rows kept (the keep smallest row losses, with a
        gap to the next one that no implementation's rounding closes)."""
        lo64 = self.old_lp(torch.float64)
        ratio = self._ratios(lp64, lo64)
        self.clip64 = (int(((ratio - 1).abs() > self.eps).sum()), int(self.mask.sum()))
        self.ratio_range = (float(ratio.min()), float(ratio.max()))
        assert 0 < self.clip64[0] < self.clip64[1], (self.clip64, self.ratio_range)        # both branches of the clipped surrogate run
        if self.keep_rows:
            rows = ppo_loss(lp64, lo64, self.tok, self.reward, SPI, self.eps, self.kl_coef, 'none')['loss']
            order = rows.sort()
            assert float(order.values[self.keep_rows] - order.values[self.keep_rows - 1]) > 1e-4 * float(rows.abs().max())
            self.kept = torch.zeros(self.N, dtype=torch.bool)
            self.kept[order.indices[:self.keep_rows]] = True

    def reference_tf32x3(self, lo=None):
        """The calibrating oracle of tc_f16x3: the fp32 oracle with every Linear's forward and input gradient as gemm_tf32 computes them,
        following float64's maxout routing; PPO's old policy is ``lo``, the old engine's own log-probs."""
        if 'g3' not in self.ref:
            rec3 = []
            loss3, lp3, g3 = self.oracle(torch.float32, route=getattr(self, 'route', None), record=rec3, tf32x3=True, lo=lo)
            self.ref.update(loss3=loss3, picked3=self.picked(lp3).double(), g3=g3)
            if self.family == 'transformer':
                self.relu_err['3xTF32 oracle'] = self._relu_err(rec3)
        return self.ref['loss3'], self.ref['picked3'], self.ref['g3']

    def _relu_err(self, rec):
        """The largest distance of an oracle's ReLU inputs from float64's, as a fraction of each layer's RMS."""
        return max(float((a.double() - a64).abs().max() / a64.pow(2).mean().sqrt()) for a, a64 in zip(rec, self.relu64))

    def _loss_l1(self, lp64):
        """(number of summed terms, sum of their magnitudes) of the step's loss."""
        if self.kind == 'ppo':
            return self.ppo_l1(lp64, self.old_lp(torch.float64))['loss']
        if self.kind in ('greedy', 'leave_one_out'):
            p = lp64.gather(2, self.tok.unsqueeze(2)).squeeze(2)
            return p.numel(), float((p * self.reward * self.mask).abs().sum() / self.mask.sum())
        if self.kind == 'autograd':
            return lp64.numel(), float((lp64 * self.G.double()).abs().sum())
        n = self.tm.numel() * (lp64.shape[2] if self.smoothing else 1)
        return n, abs(self.ref['loss64'])        # NLL and KL terms are all >= 0

    def ppo_l1(self, lp, lo):
        """{'loss' | 'pg_loss' | 'kl_loss': (number of summed terms, sum of their magnitudes)} of PPO's criterion on the log-probs lp, lo
        (a position's KL term is itself a sum over the vocabulary)."""
        m, idx = self.mask, self.tok.unsqueeze(2)
        ratio = torch.exp(lp.gather(2, idx) - lo.gather(2, idx)).squeeze(2)
        adv = self.adv.unsqueeze(1)
        pg = torch.maximum(-adv * ratio, -adv * ratio.clamp(1 - self.eps, 1 + self.eps)).abs() * m
        kl = (lo.exp() * (lo - lp)).abs().sum(2) * m
        total = m.sum()
        w = self.kept.double().unsqueeze(1) / (m.sum(1, keepdim=True) * self.keep_rows) if self.keep_rows else 1 / total
        n_pg, n_kl = int(total), int(total) * lp.shape[2]
        return {'loss': (n_pg + n_kl, float(((pg + self.kl_coef * kl) * w).sum())), 'pg_loss': (n_pg, float(pg.sum() / total)),
                'kl_loss': (n_kl, float(kl.sum() / total))}

    def maxout_delta(self, unit, bases):
        """float64 gradient change of re-routing one maxout unit (t, n, j): only caption row n's share of the loss changes.  ``bases`` caches
        each row's share as float64 routes it."""
        t, n, j = unit
        route = [r[[n, n]] for r in self.route]
        if n not in bases:
            bases[n] = self.oracle(torch.float64, rows=n, route=route)[2]
        base = bases[n]
        flip = torch.zeros(2, self.c['H'], dtype=torch.bool)
        flip[0, j] = True
        _, _, moved = self.oracle(torch.float64, rows=n, route=route, flip={t: flip})
        return {k: moved[k] - base[k] for k in base}


def _fit_maxout(case, named):
    """The float64 gradients with each ambiguous maxout unit routed the way that fits the engine better; returns (gradients, re-routed)."""
    g64 = {k: v.clone() for k, v in case.ref['g64'].items()}
    largest = max(float(v.abs().max()) for v in g64.values())
    scale = {k: float(v.abs().max()) + 1e-6 * largest for k, v in g64.items()}       # a zero-gradient tensor's noise must not decide
    keep = {k: case.keep.get(k, torch.ones((), dtype=torch.bool)) for k in g64}          # ReLU kink entries say nothing about the maxout
    moved, bases = 0, {}
    for u in case.maxout:
        delta = case.maxout_delta(u, bases)

        def miss(k, d):
            return float((((named[k].double() - g64[k] - d) / scale[k]) * keep[k]).pow(2).sum())
        before = sum(miss(k, 0.0) for k in delta)
        after = sum(miss(k, delta[k]) for k in delta)
        size = sum(float(((delta[k] / scale[k]) * keep[k]).pow(2).sum()) for k in delta)
        # after - before = size - 2 <misfit, delta>: the engine's misfit must project onto delta at ~0 (not re-routed) or ~1 (re-routed),
        # never in between, so an engine error can never pass for a maxout decision
        assert size < 1e-18 or abs(after - before) >= 0.8 * size, (u, before, after, size)
        if after < before:
            for k in delta:
                g64[k] += delta[k]
            moved += 1
    return g64, moved


def _scalar_bar(err, floor=1e-6, factor=4.0):
    return max(factor * err, floor)


def _sum_floor(n, l1):
    """The pairwise-summation bound 2^-24 x log2(terms) x sum of |terms| of a sum reduced in another order than torch's (at least 1e-6)."""
    return max(1e-6, 2.0 ** -24 * np.log2(n) * l1)


def _check_ppo(label, case, got):
    """PPO's old policy and criterion: the old engine's log-probs held to float64 at every position the mask keeps; the engine's clipfrac
    equal, as an fp32 value, to float64's clip count over the mask sum; and loss, pg_loss, kl_loss and clipfrac recomputed in float64 from
    the engine's own new and old log-probs and scores, within the summation bound (ppo_mask / row / reduce_kernel alone, apart from the
    model's arithmetic)."""
    keep = case.mask > 0
    lo64 = case.old_lp(torch.float64)
    e_lo = float((got['lo'].double() - lo64).abs().amax(2)[keep].max())
    print('%s cliprange %g: clipfrac %d / %d, ratios %.3g .. %.3g; old policy log-probs err %.2e' % (
        label, case.eps, case.clip64[0], case.clip64[1], case.ratio_range[0], case.ratio_range[1], e_lo))
    assert e_lo < LOGP_TOL, e_lo
    n_clip, total = case.clip64
    assert got['stats']['clipfrac'] == float(torch.tensor(n_clip / total, dtype=torch.float32)), (got['stats']['clipfrac'], n_clip, total)
    lp, lo = got['lp'].double(), got['lo'].double()
    out = ppo_loss(lp, lo, case.tok, got['reward'].double(), SPI, case.eps, case.kl_coef, 'none' if case.keep_rows else 'mean')
    if case.keep_rows:
        out['loss'] = out['loss'].sort().values[:case.keep_rows].mean()
    l1 = case.ppo_l1(lp, lo)
    for k in ('loss', 'pg_loss', 'kl_loss', 'clipfrac'):
        e = abs(got['stats'][k] - float(out[k]))
        bar = _sum_floor(*l1[k]) if k in l1 else 2.0 ** -24       # clipfrac: a count over the mask sum, one rounding
        print('%s criterion %s %.6g err %.2e bar %.2e' % (label, k, float(out[k]), e, bar))
        assert e <= bar, (k, e, bar)


def _reference(family, kind, dropout, B, smoothing, regions, masks_fn, modes, ppo=None):
    key = (family, kind, dropout, B, smoothing, regions, ppo)
    if key not in _CASES:
        case = Case(family, kind, dropout, B, smoothing, regions, ppo)
        if dropout:
            case.drop = masks_fn(case)
        case.reference()
        case.uses = 0
        _CASES[key] = case
    case = _CASES[key]
    case.uses += 1
    if case.uses == modes:                # every mode this case runs in has had it
        del _CASES[key]
    return case


def _masks_fn(family):
    import imagecaptioning.pytorch_b200 as b200

    def make(case):
        c, steps = case.c, case.steps
        if family == 'aoa':
            return aoa_masks(b200, SEED, case.B, case.Rc, case.N, steps, c['E'], c['H'], HEADS, *RATES['aoa'])
        if family == 'transformer':
            return tfm_masks(b200, SEED, case.B, case.Rc, case.N, steps, T, c['E'], c['H'], HEADS, c['A'], *RATES['transformer'])
        if family == 'newfc':               # its one site, the core output (UpDown's site 3)
            return {'out': dropout_masks(b200, SEED, RATES[family], case.B, 1, case.N, steps, c['E'], c['H'])['out']}
        fn = dropout_masks if family == 'updown' else att2in2_masks
        return fn(b200, SEED, RATES[family], case.B, case.Rc, case.N, steps, c['E'], c['H'])
    return make


def _check_masks(family, drop):
    if family == 'transformer':         # drop_prob_lm at att_embed, the Transformer's own rate at every other site
        rates = {k: RATES[family][0] if k == 'att_embed' else RATES[family][1] for k in drop}
    else:
        rates = RATES[family] if family == 'aoa' else (RATES[family],) * 4
        rates = {k: rates[1] if k.startswith('ref_p') or k == 'p' else rates[2] if k.startswith('ref_aoa') else rates[3] if k.startswith('ref_sub')
                 else rates[0] for k in drop}
    for k, m in drop.items():
        p = rates[k]
        assert abs(float((m > 0).double().mean()) - (1 - p)) < 0.02, (k, p)


def _run_engine(family, mode, case):
    model = _model(family, mode, autograd=case.kind == 'autograd')
    if family == 'transformer':
        model.load_state_dict(case.W, strict=True)            # this case's weights, off the ReLU kinks
    fc, att = case.fc.cuda(), case.att.cuda()
    reg = None if case.regions is None else case.regions.cuda()
    if family == 'aoa':
        p = RATES['aoa'] if case.dropout else (0.0,) * 4
        rates = dict(drop_prob=p[0], drop_attn=p[1], drop_aoa=p[2], drop_sublayer=p[3], ctx_drop=1)
    elif family == 'transformer':
        p = RATES['transformer'] if case.dropout else (0.0, 0.0)
        rates = dict(drop_prob=p[0], dropout=p[1])
    else:
        rates = dict(drop_prob=RATES[family] if case.dropout else 0.0)
    name_of = {id(p): k for k, p in model.state_dict(keep_vars=True).items()}
    if case.kind == 'autograd':
        model.eval()
        for p in model.parameters():
            p.grad = None
        lp = model(fc, att, case.labels[..., :-1].cuda(), reg)
        (lp * case.G.cuda()).sum().backward()
        torch.cuda.synchronize()
        return dict(lp=lp.detach().cpu(),
                    grads={k: p.grad.detach().cpu() for k, p in model.state_dict(keep_vars=True).items() if isinstance(p, torch.nn.Parameter)})
    model.train()
    extra = {}
    if case.kind == 'xe':
        res = model.xe_step(fc, att, case.labels.cuda(), case.lmasks.cuda(), label_smoothing=case.smoothing, seed=SEED, att_masks=reg, **rates)
        lp = res['logprobs']
    elif case.kind == 'ppo':
        import imagecaptioning.pytorch_b200 as b200
        old = _model(family, mode, old=True)
        old.load_state_dict(case.W_old, strict=True)
        old.eval()
        res = model.ppo_step(old, fc, att, case.gts, b200.rewards.CiderDTable(case.df, case.ref_len), SPI, cliprange=case.eps,
                             kl_coef=case.kl_coef, seed=SEED, forced_tokens=case.tok.cuda(), att_masks=reg, keep_rows=case.keep_rows, **rates)
        assert torch.equal(res['sample_seq'].cpu(), case.tok)
        lp = res['sample_logprobs']
        # the old engine's own eval-mode teacher-forced pass: what the step's old pass computes (the same teacher path)
        with torch.no_grad():
            lo = old(fc, att, old_policy_input(case.tok).cuda(), reg).float().cpu()
        if lo.shape[1] < T:             # stopped where every row had ended: those positions are all masked
            lo = torch.nn.functional.pad(lo, (0, 0, 0, T - lo.shape[1]))
        extra = dict(lo=lo, reward=res['scores'].detach().cpu().view(-1), stats={k: float(res[k]) for k in ('loss', 'pg_loss', 'kl_loss', 'clipfrac')})
    else:
        import imagecaptioning.pytorch_b200 as b200
        table = b200.rewards.CiderDTable(case.df, case.ref_len)
        kw = dict(forced_tokens=case.tok.cuda(), att_masks=reg, seed=SEED, **rates)
        if case.kind == 'greedy':
            res = model.scst_step(fc, att, case.gts, table, SPI, forced_baseline=case.base.cuda(), **kw)
            assert torch.equal(res['greedy_seq'].cpu(), case.base)
        else:
            res = model.scst_step(fc, att, case.gts, table, SPI, baseline='leave_one_out', **kw)
        assert torch.equal(res['sample_seq'].cpu(), case.tok)
        lp = res['sample_logprobs']
    torch.cuda.synchronize()
    out = dict(loss=float(res['loss']), lp=lp.detach().cpu(), grads={name_of[id(p)]: g.detach().cpu() for p, g in res['grads'].items()})
    if case.kind in ('greedy', 'leave_one_out'):
        out['reward'] = res['reward'].detach().cpu()
    out.update(extra)
    return out


def _compare(family, mode, case):
    t0 = time.time()
    got = _run_engine(family, mode, case)
    ref = case.ref
    if mode == 'tc_f16x3':
        loss_c, picked_c, g_c = case.reference_tf32x3(got.get('lo'))
        oname, factor = '3xTF32 oracle', 4.0
    else:
        loss_c, picked_c, g_c = ref['loss32'], ref['picked32'], ref['g32']
        oname, factor = 'fp32 oracle', 4.0
    kind = case.kind + (' ls=%g' % case.smoothing if case.kind == 'xe' else '')
    if case.kind == 'ppo':
        kind += ' perturb=%g kl=%g keep=%d' % (case.perturb, case.kl_coef, case.keep_rows)
    label = '[%s %s %s drop=%s N=%d%s]' % (family, mode, kind, case.dropout, case.N, ' regions' if case.regions is not None else '')
    print('%s float64 reference %.1f s; ReLU units left out per layer %s, %d ambiguous maxout units' % (label, case.ref_seconds, case.kink_rows,
                                                                                                       len(case.maxout)))
    if case.kind == 'ppo':
        _check_ppo(label, case, got)
    assert all(v <= 0.15 * case.c["H"] for v in case.kink_rows.values()), case.kink_rows        # some rows of the layer, not the layer
    if family == 'transformer':
        print('%s ReLU units shifted per layer %s; largest shift %.2e x RMS' % (label, case.shifted, case.largest_shift))
        err = case.relu_err[oname]
        print('%s ReLU inputs clear of their kinks by %.1e x RMS; %s error there %.2e x RMS (5x = %.2f of the margin)' % (
            label, TFM_MARGIN, oname, err, 5 * err / TFM_MARGIN))
        assert 5 * err < TFM_MARGIN, (oname, err)
        assert len(got['grads']) == 261, len(got['grads'])             # every parameter (pe is a buffer)
    if family == 'newfc':
        assert len(got['grads']) == 9, len(got['grads'])
    # scalars: loss (not for the autograd case, whose objective is a sum over every log-prob), picked log-probs, reward
    if 'loss' in got:
        n, l1 = ref['l1']
        floor = max(1e-6, 2.0 ** -24 * np.log2(n) * l1)
        ec = abs(loss_c - ref['loss64'])
        e = abs(got['loss'] - ref['loss64'])
        print('%s loss %.6f err %.2e bar %.2e (%s %.2e)' % (label, ref['loss64'], e, _scalar_bar(ec, floor, factor), oname, ec))
        assert e <= _scalar_bar(ec, floor, factor), ('loss', e, ec, floor)
        assert abs(ref['loss64']) > 1e-3 or case.kind in ('leave_one_out', 'ppo')
    picked = case.picked(got['lp']).double()
    ec = float((picked_c - ref['picked64']).abs().max())
    e = float((picked - ref['picked64']).abs().max())
    print('%s picked log-probs err %.2e bar %.2e (%s %.2e)' % (label, e, _scalar_bar(ec, 1e-6, factor), oname, ec))
    assert e <= _scalar_bar(ec, 1e-6, factor), ('picked log-probs', e, ec)
    if 'reward' in got:
        ec = float((case.reward.float().double() - case.reward).abs().max())
        e = float((got['reward'].double() - case.reward).abs().max())
        assert e <= _scalar_bar(ec, 1e-6, factor), ('reward', e, ec)
        assert float(case.reward.abs().max()) > 1e-2
    # gradients; the float64 side re-routed at the ambiguous maxout units the way the engine went
    g64, moved = (_fit_maxout(case, got['grads']) if case.maxout else (ref['g64'], 0))
    if case.maxout:
        print('%s maxout units re-routed to fit the engine: %d of %d' % (label, moved, len(case.maxout)))
    # the fp32 oracle followed float64's routing: it is measured against the float64 gradients before the re-routing
    gc = {k: g_c[k].double() + (g64[k] - ref['g64'][k]) for k in g64}
    # a weight gradient reduces over every (step, row) pair; rounding of a sequential fp32 accumulation grows as the square root of that
    # length (simt_fp32's gemm_wgrad_launch: core.lang_lstm.weight_ih measured at 0.43 / 0.62 / 1.03 of the fixed 2e-6 floor for 1000 / 3200
    # / 6400 pairs), so the floor does.  In tc_f16x3 the calibrating oracle's own error is the larger term.
    floor = 2e-6 * max(1.0, case.N * case.steps / 1000) ** 0.5
    worst = check_grads_f64(got['grads'], g64, gc, keep=case.keep, label=label, floor=floor, factor=factor)
    print('%s worst gradient err/bar %.3f; compared in %.1f s' % (label, worst, time.time() - t0))


MODES = ['tc_f16x3', 'simt_fp32']
STEPS = [('greedy', 0.0), ('leave_one_out', 0.0), ('xe', 0.0), ('xe', 0.1)]


# the modes each family runs in (see the module docstring on Att2in2 in tc_f16x3)
FAMILY_MODES = {'updown': MODES, 'att2in2': ['simt_fp32'], 'newfc': MODES, 'aoa': MODES, 'transformer': MODES}


def _run(family, mode, kind, smoothing, dropout, B, regions=None, ppo=None):
    regions = kind == 'leave_one_out' if regions is None else regions
    case = _reference(family, kind, dropout, B, smoothing, regions, _masks_fn(family), len(FAMILY_MODES[family]), ppo)
    if dropout:
        _check_masks(family, case.drop)
    _compare(family, mode, case)


@pytest.mark.parametrize('dropout', [False, True])
@pytest.mark.parametrize('kind,smoothing', STEPS)
@pytest.mark.parametrize('mode', MODES)
def test_updown_step_f64(mode, kind, smoothing, dropout):
    _run('updown', mode, kind, smoothing, dropout, 10)


@pytest.mark.parametrize('B', [32, pytest.param(64, marks=pytest.mark.slow)])
@pytest.mark.parametrize('kind,smoothing', [('greedy', 0.0), ('xe', 0.1)])
@pytest.mark.parametrize('mode', MODES)
def test_updown_step_f64_rows(mode, kind, smoothing, B):
    """160 and 320 rows per step.  In tc_f16x3 the per-step GEMMs run gemm_tf32's swapped tile of width 256 (160 rows) and its normal
    orientation (320 rows); in simt_fp32 the same steps at larger M through gemm_generic."""
    _run('updown', mode, kind, smoothing, True, B)


@pytest.mark.parametrize('dropout', [False, True])
@pytest.mark.parametrize('kind,smoothing', STEPS)
@pytest.mark.parametrize('mode', ['simt_fp32'])
def test_att2in2_step_f64(mode, kind, smoothing, dropout):
    """simt_fp32 only: see the module docstring on Att2in2's maxout in tc_f16x3."""
    _run('att2in2', mode, kind, smoothing, dropout, 10)


@pytest.mark.parametrize('dropout', [False, True])
@pytest.mark.parametrize('kind,smoothing', STEPS)
@pytest.mark.parametrize('mode', MODES)
def test_aoa_step_f64(mode, kind, smoothing, dropout):
    _run('aoa', mode, kind, smoothing, dropout, 10)


@pytest.mark.parametrize('dropout', [False, True])
@pytest.mark.parametrize('kind,smoothing', STEPS)
@pytest.mark.parametrize('mode', MODES)
def test_transformer_step_f64(mode, kind, smoothing, dropout):
    _run('transformer', mode, kind, smoothing, dropout, 10)


@pytest.mark.slow
@pytest.mark.parametrize('kind,smoothing', [('greedy', 0.0), ('xe', 0.1)])
@pytest.mark.parametrize('mode', MODES)
def test_transformer_step_f64_rows(mode, kind, smoothing):
    """160 rows per step: in tc_f16x3 the per-position GEMMs of the sampled pass run gemm_tf32's swapped tile of width 256, and the
    batched backward runs over 160 x 21 = 3360 rows."""
    _run('transformer', mode, kind, smoothing, True, 32)


@pytest.mark.parametrize('family,mode', [(f, m) for f in ('updown', 'att2in2', 'aoa', 'transformer') for m in MODES
                                         if (f, m) != ('att2in2', 'tc_f16x3')])
def test_autograd_teacher_f64(family, mode):
    """model.autograd: teacher-forced log-probs under grad and the backward of a seeded upstream gradient (logsoftmax_vjp_kernel<4>:
    V + 1 = 9488 is a multiple of 4)."""
    case = _reference(family, 'autograd', False, 10, 0.0, True, None, 1 if family == 'att2in2' else len(MODES))
    _compare(family, mode, case)


@pytest.mark.parametrize('dropout', [False, True])
@pytest.mark.parametrize('kind,smoothing', STEPS)
@pytest.mark.parametrize('mode', FAMILY_MODES['newfc'])
def test_newfc_step_f64(mode, kind, smoothing, dropout):
    """NewFC at the fc_rl / fc_nsc recipe width (E = H = 512, F_fc 2048); its core is co.maxout_lstm, so its ambiguous maxout units are
    re-routed to fit the engine as Att2in2's.  It reads no region features: no case has region masks."""
    _run('newfc', mode, kind, smoothing, dropout, 10, regions=False)


@pytest.mark.parametrize('mode', FAMILY_MODES['newfc'])
def test_newfc_autograd_teacher_f64(mode):
    """test_autograd_teacher_f64 for NewFC, without region masks."""
    case = _reference('newfc', 'autograd', False, 10, 0.0, False, None, len(FAMILY_MODES['newfc']))
    _compare('newfc', mode, case)


# PPO cases: (old-policy perturbation, kl_coef, keep_rows, dropout, region masks)
PPO_CASES = {'old_equals_new': (False, KL_COEF, 0, True, False),
             'perturbed': (True, KL_COEF, 0, False, False),
             'regions': (True, KL_COEF, 0, False, True),
             'kl_coef_1': (True, KL_COEF_FULL, 0, False, False),
             'keep_rows': (True, KL_COEF, PPO_KEEP, False, False)}


def _ppo_params():
    out = []
    for f, modes in FAMILY_MODES.items():
        for c in PPO_CASES:
            # Att2in2 without region masks: with perturbed old weights fewer than 15 of its gradient tensors reach 1e-5, check_grads_f64's
            # floor for a comparison that says something, so its perturbed cases run with region masks (kl_coef_1 included)
            if (c == 'regions' and f == 'newfc') or (c == 'keep_rows' and f != 'updown') or (f == 'att2in2' and c == 'perturbed'):
                continue
            for m in modes:         # a case's modes in a row: its references are freed after the last
                slow = m == 'tc_f16x3' and c in ('regions', 'kl_coef_1')           # the same paths as the mode's other cases
                out.append(pytest.param(f, m, c, marks=pytest.mark.slow) if slow else (f, m, c))
    return out


@pytest.mark.parametrize('family,mode,case', _ppo_params())
def test_ppo_step_f64(family, mode, case):
    """ppo_step: the new policy's sampled pass (samples replayed), the old policy's eval-mode teacher-forced pass over [0, samples[:, :-1]],
    the leave-one-out advantage of the CIDEr-D scores and the clipped-ratio + KL criterion, against float64 with the backward through the
    new policy only.  old_equals_new: the old policy holds the new weights and the ratios move by the new policy's dropout (recipe rates)
    alone; the others perturb the old weights, without dropout."""
    perturbed, kl_coef, keep, dropout, regions = PPO_CASES[case]
    regions = regions or (family == 'att2in2' and perturbed)
    _run(family, mode, 'ppo', 0.0, dropout, 10, regions=regions, ppo=(PERTURB[family] if perturbed else 0.0, kl_coef, keep))
