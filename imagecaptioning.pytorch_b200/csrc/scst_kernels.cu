// Kernels of the SCST training step that have no counterpart in decoding: replayable dropout, the backward of
// log-softmax + RewardCriterion, nn.LSTMCell, additive attention, ReLU/dropout, the embedding scatter and per-image sums.
//
// What they differentiate (reference, relative to /root/reference/captioning):
//   dropout sites            models/AttModel.py:74-88 (embed / fc_embed / att_embed Sequentials), :637 (core output)
//   dlogits                  modules/losses.py:22-37 (RewardCriterion) composed with F.log_softmax (AttModel.py:172)
//   lstm_cell_backward       nn.LSTMCell (AttModel.py:628,635)
//   maxout_cell_backward     Att2in2Core's maxout cell (AttModel.py:773-787) and NewFC's LSTMCore (FCModel.py:25-42)
//   attention_backward       models/AttModel.py:728-748
//   ppo                      modules/losses.py:267-357 (PPOLoss) composed with F.log_softmax
// Dropout masks are never stored: keep(seed, site, step, element) is a pure function (Philox4x32-10), re-evaluated in the backward.
#include <type_traits>

#include "common.cuh"
#include "dropout.cuh"
#include "kernels.cuh"

namespace capb200 {

namespace {

__global__ void dropout_apply_kernel(float* x, long n, int cols, long ld, unsigned long long seed, uint32_t site, uint32_t step, float p) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const long r = i / cols;
        const int c = (int)(i % cols);
        x[r * ld + c] *= drop_scale(seed, site, step, (uint32_t)i, p);
    }
}

__global__ void dropout_mask_kernel(float* m, long n, unsigned long long seed, uint32_t site, uint32_t step, float p) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) m[i] = drop_scale(seed, site, step, (uint32_t)i, p);
}

// y[r, c] = x[r, c] * dropmask(site, step, r*cols + c)  with separate pitches (core output -> [N, T, H] tape slot)
__global__ void dropout_copy_kernel(const float* __restrict__ x, long ld_x, float* __restrict__ y, long ld_y, int rows, int cols, unsigned long long seed,
                                    uint32_t site, uint32_t step, float p) {
    const long n = (long)rows * cols;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const long r = i / cols;
        const int c = (int)(i % cols);
        y[r * ld_y + c] = x[r * ld_x + c] * drop_scale(seed, site, step, (uint32_t)i, p);
    }
}

// xt[r, :] = relu(emb[tok[r], :]) * dropmask
__global__ void embed_relu_dropout_kernel(int rows, int E, const int* __restrict__ tokens, const float* __restrict__ emb, float* __restrict__ xt,
                                          unsigned long long seed, uint32_t step, float p) {
    const int r = blockIdx.x;
    const float* e = emb + (long)tokens[r] * E;
    for (int c = threadIdx.x; c < E; c += blockDim.x) xt[(long)r * E + c] = fmaxf(__ldg(e + c), 0.f) * drop_scale(seed, 2u, step, (uint32_t)(r * E + c), p);
}

// d logits of  loss = sum_{n,t} -logp[n,t,seq] * reward[n] * mask[n,t] / sum(mask)  through log_softmax:
//   dl[n,t,v] = coef * (1[v == seq] - exp(logp[n,t,v])),  coef = -reward[n,t] * mask[n,t] / mask_sum * upstream
__global__ void scst_dlogits_kernel(const float* __restrict__ logp, long ld_row, const long long* __restrict__ seq, const float* __restrict__ reward,
                                    const float* __restrict__ mask_sum, float upstream, int T, int V1, float* __restrict__ dl,
                                    const float* __restrict__ row_coef) {
    const long item = blockIdx.x;                 // n * T + t
    const int t = (int)(item % T);
    const long n = item / T;
    const float m = (t == 0 || seq[n * T + t - 1] > 0) ? 1.f : 0.f;
    // reduction 'mean': upstream / (all mask entries); drop_worst: upstream / (k * this row's mask entries) for kept rows, 0 for dropped ones
    const float coef = -reward[item] * m * (row_coef != nullptr ? row_coef[n] : upstream / (*mask_sum));
    const long long tok = seq[item];
    const float* lp = logp + n * ld_row + (long)t * V1;
    float* d = dl + item * V1;
    if (coef == 0.f) {
        for (int v = threadIdx.x; v < V1; v += blockDim.x) d[v] = 0.f;
        return;
    }
    for (int v = threadIdx.x; v < V1; v += blockDim.x) d[v] = coef * ((v == tok ? 1.f : 0.f) - expf(lp[v]));
}

// Backward of log_softmax for an outside gradient G = dL/dlogp: dl[n,t,v] = G[n,t,v] - exp(logp[n,t,v]) * sum_v' G[n,t,v'].  One CTA per
// (n, t), VEC floats per load.  With `seq` (sampling form) a row that had finished before step t was written as zeros by the forward
// (AttModel.py:341: logprobs * unfinished), so its d logits are zero.
template <int VEC>
__global__ void __launch_bounds__(256) logsoftmax_vjp_kernel(const float* __restrict__ logp, const float* __restrict__ g, long ld_row,
                                                             const long long* __restrict__ seq, int T, int V1, float* __restrict__ dl) {
    using V = typename std::conditional<VEC == 4, float4, float>::type;
    __shared__ float red[32];
    const long item = blockIdx.x;                 // n * T + t
    const int t = (int)(item % T);
    const long n = item / T;
    const int nv = V1 / VEC;
    V* d = reinterpret_cast<V*>(dl + item * V1);
    if (seq != nullptr && t > 0 && seq[n * T + t - 1] == 0) {
        const V z = {};
        for (int i = threadIdx.x; i < nv; i += blockDim.x) d[i] = z;
        return;
    }
    const V* gr = reinterpret_cast<const V*>(g + n * ld_row + (long)t * V1);
    const V* lr = reinterpret_cast<const V*>(logp + n * ld_row + (long)t * V1);
    auto hsum = [](const V& x) {
        if constexpr (VEC == 4) return (x.x + x.y) + (x.z + x.w);
        else return x;
    };
    float s = 0.f;
    for (int i = threadIdx.x; i < nv; i += blockDim.x) s += hsum(gr[i]);
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 32) {
        s = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (threadIdx.x == 0) red[0] = s;
    }
    __syncthreads();
    s = red[0];
    for (int i = threadIdx.x; i < nv; i += blockDim.x) {
        const V gv = gr[i], lv = lr[i];
        V o;
        if constexpr (VEC == 4) o = make_float4(gv.x - expf(lv.x) * s, gv.y - expf(lv.y) * s, gv.z - expf(lv.z) * s, gv.w - expf(lv.w) * s);
        else o = gv - expf(lv) * s;
        d[i] = o;
    }
}

// ---- cross-entropy stage (LanguageModelCriterion / LabelSmoothing, losses.py:204-265) on teacher-forced log-probs [N, Ls, V1]:
// target[n, t] = labels[n, t + 1], mask[n, t] = masks[n, t + 1]; steps <= Ls columns were evaluated (the rest stay zero, AttModel.py:158-159).
__global__ void xe_mask_sum_kernel(const float* __restrict__ masks, long ld_m, int N, int Ls, float* __restrict__ mask_sum) {
    __shared__ float sh[256];
    float s = 0.f;
    for (int i = threadIdx.x; i < N * Ls; i += 256) s += masks[(long)(i / Ls) * ld_m + (i % Ls) + 1];
    sh[threadIdx.x] = s;
    __syncthreads();
    for (int w = 128; w > 0; w >>= 1) {
        if (threadIdx.x < w) sh[threadIdx.x] += sh[threadIdx.x + w];
        __syncthreads();
    }
    if (threadIdx.x == 0) *mask_sum = sh[0];
}

// one CTA per (n, t < steps): d logits = coef * (softmax - target_dist), coef = mask / mask_sum * upstream; item_loss = un-normalised loss term
__global__ void __launch_bounds__(256) xe_dlogits_kernel(const float* __restrict__ logp, long ld_row, const long long* __restrict__ labels, long ld_l,
                                                         const float* __restrict__ masks, long ld_m, const float* __restrict__ mask_sum, float upstream,
                                                         float smoothing, int steps, int V1, float* __restrict__ dl, float* __restrict__ item_loss,
                                                         const float* __restrict__ row_coef) {
    __shared__ float sh[256];
    const long item = blockIdx.x;                 // n * steps + t
    const int t = (int)(item % steps);
    const long n = item / steps;
    const float m = masks[n * ld_m + t + 1];
    const long long tgt = labels[n * ld_l + t + 1];
    const float coef = m * (row_coef != nullptr ? row_coef[n] : upstream / (*mask_sum));
    const float* lp = logp + n * ld_row + (long)t * V1;
    float* d = dl + item * V1;
    const float off = smoothing > 0.f ? smoothing / (float)(V1 - 1) : 0.f, conf = 1.f - smoothing;
    float lsum = 0.f;
    for (int v = threadIdx.x; v < V1; v += 256) {
        const float l = lp[v];
        const float td = (v == tgt) ? conf : off;
        d[v] = coef * (expf(l) - td);
        if (smoothing > 0.f) lsum += (td > 0.f) ? td * (logf(td) - l) : 0.f;           // KLDivLoss pointwise term (xlogy convention)
    }
    sh[threadIdx.x] = lsum;
    __syncthreads();
    for (int w = 128; w > 0; w >>= 1) {
        if (threadIdx.x < w) sh[threadIdx.x] += sh[threadIdx.x + w];
        __syncthreads();
    }
    if (threadIdx.x == 0) item_loss[item] = (smoothing > 0.f ? sh[0] : -lp[tgt]) * m;
}

// loss = (sum of item terms + the terms of the never-evaluated columns, whose log-probs are zero) / mask_sum
__global__ void xe_loss_kernel(const float* __restrict__ item_loss, int N, int steps, int Ls, const float* __restrict__ masks, long ld_m, float smoothing,
                               int V1, const float* __restrict__ mask_sum, float* __restrict__ loss) {
    __shared__ float sh[256];
    float s = 0.f;
    for (int i = threadIdx.x; i < N * steps; i += 256) s += item_loss[i];
    if (smoothing > 0.f && steps < Ls) {
        const float off = smoothing / (float)(V1 - 1), conf = 1.f - smoothing;
        const float zero_row = (float)(V1 - 1) * off * logf(off) + (conf > 0.f ? conf * logf(conf) : 0.f);
        const int extra = Ls - steps;
        for (int i = threadIdx.x; i < N * extra; i += 256) s += zero_row * masks[(long)(i / extra) * ld_m + steps + (i % extra) + 1];
    }
    sh[threadIdx.x] = s;
    __syncthreads();
    for (int w = 128; w > 0; w >>= 1) {
        if (threadIdx.x < w) sh[threadIdx.x] += sh[threadIdx.x + w];
        __syncthreads();
    }
    if (threadIdx.x == 0) *loss = sh[0] / (*mask_sum);
}

// ---- drop_worst (tools/train.py:187-191): the criterion runs with reduction 'none' (one loss per caption row, normalised by that row's mask
// entries) and the trainer averages the k rows with the SMALLEST loss.  The selection happens on the device between the forward and the
// backward of the fused step: row_coef[n] = upstream / (k * row_mask[n]) for kept rows, 0 for dropped ones; loss = mean over the kept rows.
__global__ void xe_row_loss_kernel(const float* __restrict__ item_loss, int N, int steps, int Ls, const float* __restrict__ masks, long ld_m, float smoothing,
                                   int V1, float* __restrict__ row_loss, float* __restrict__ row_msum) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    float s = 0.f, ms = 0.f;
    for (int t = 0; t < steps; ++t) s += item_loss[(long)n * steps + t];
    for (int t = 0; t < Ls; ++t) ms += masks[(long)n * ld_m + t + 1];
    if (smoothing > 0.f && steps < Ls) {          // never-evaluated columns: their log-prob rows are zero (AttModel.py:158-159)
        const float off = smoothing / (float)(V1 - 1), conf = 1.f - smoothing;
        const float zero_row = (float)(V1 - 1) * off * logf(off) + (conf > 0.f ? conf * logf(conf) : 0.f);
        for (int t = steps; t < Ls; ++t) s += zero_row * masks[(long)n * ld_m + t + 1];
    }
    row_loss[n] = s / ms;
    row_msum[n] = ms;
}

__global__ void scst_row_mask_kernel(const long long* __restrict__ seq, int N, int T, float* __restrict__ row_msum) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    float ms = 0.f;
    for (int t = 0; t < T; ++t) ms += (t == 0 || seq[(long)n * T + t - 1] > 0) ? 1.f : 0.f;
    row_msum[n] = ms;
}

// single CTA: rank every row among all rows (ties: lower index first), keep the k smallest
__global__ void __launch_bounds__(256) drop_worst_select_kernel(const float* __restrict__ row_loss, const float* __restrict__ row_msum, int N, int k,
                                                                float upstream, float* __restrict__ row_coef, float* __restrict__ loss) {
    __shared__ float sh[256];
    float acc = 0.f;
    for (int n = threadIdx.x; n < N; n += 256) {
        const float l = row_loss[n];
        int rank = 0;
        for (int j = 0; j < N; ++j) {
            const float lj = row_loss[j];
            rank += (lj < l || (lj == l && j < n)) ? 1 : 0;
        }
        const bool kept = rank < k;
        row_coef[n] = kept ? upstream / ((float)k * row_msum[n]) : 0.f;
        if (kept) acc += l;
    }
    sh[threadIdx.x] = acc;
    __syncthreads();
    for (int w = 128; w > 0; w >>= 1) {
        if (threadIdx.x < w) sh[threadIdx.x] += sh[threadIdx.x + w];
        __syncthreads();
    }
    if (threadIdx.x == 0) *loss = sh[0] / (float)k;
}

// ---- PPO (losses.py:267-357): the clipped policy-ratio loss against a frozen old policy plus a token-level KL penalty.
// lp [N, T, V1] are the new policy's sampled log-probs, lo [N, T, V1] the old policy's teacher-forced ones over the same words,
// mask[n, t] = 1 for t = 0 or seq[n, t-1] > 0.
// The old policy's input words: [0, seq[:, :-1]] (losses.py:319)
__global__ void ppo_shift_kernel(const long long* __restrict__ seq, int N, int T, long long* __restrict__ tokens_in) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N * T) return;
    const int t = i % T;
    tokens_in[i] = t == 0 ? 0 : seq[i - 1];
}

// single CTA: each row's mask count and their total
__global__ void __launch_bounds__(256) ppo_mask_kernel(const long long* __restrict__ seq, int N, int T, float* __restrict__ row_msum,
                                                       float* __restrict__ mask_sum) {
    __shared__ float sh[256];
    float acc = 0.f;
    for (int n = threadIdx.x; n < N; n += 256) {
        float ms = 0.f;
        for (int t = 0; t < T; ++t) ms += (t == 0 || seq[(long)n * T + t - 1] > 0) ? 1.f : 0.f;
        row_msum[n] = ms;
        acc += ms;
    }
    sh[threadIdx.x] = acc;
    __syncthreads();
    for (int w = 128; w > 0; w >>= 1) {
        if (threadIdx.x < w) sh[threadIdx.x] += sh[threadIdx.x + w];
        __syncthreads();
    }
    if (threadIdx.x == 0) *mask_sum = sh[0];
}

// One CTA per (n, t).  ratio = exp(lp[seq] - lo[seq]); pg = max(-adv ratio, -adv clamp(ratio, 1 - eps, 1 + eps)); kl = sum_v exp(lo) (lo - lp)
// (F.kl_div(lp, lo, log_target=True)); clip = |ratio - 1| > eps.  The gradient G = d loss / d lp of the row, scaled by coef:
//   at the picked word  -adv ratio when the unclamped branch is taken (inside the clip range torch.maximum splits the gradient between two
//                       equal branches whose sum is that), 0 when the clamped one is larger;
//   on every word       -kl_coef exp(lo_v);
// and the log-softmax backward folded in: dl = G - exp(lp) sum(G).  coef = mask * upstream / sum(mask) (reduction 'mean'), or mask alone for
// drop_worst, whose per-row coefficient is applied after the selection (ppo_scale_rows_kernel).  terms [3][N*T]: masked pg, kl, clip.
__global__ void __launch_bounds__(256) ppo_row_kernel(const float* __restrict__ lp, long ld_lp, const float* __restrict__ lo, const long long* __restrict__ seq,
                                                      const float* __restrict__ adv, const float* __restrict__ mask_sum, float upstream, bool per_row,
                                                      float eps, float kl_coef, int T, int V1, float* __restrict__ dl, float* __restrict__ terms) {
    __shared__ float red[2][32];
    const long item = blockIdx.x;                 // n * T + t
    const long NT = (long)gridDim.x;
    const int t = (int)(item % T);
    const long n = item / T;
    float* d = dl + item * V1;
    const float m = (t == 0 || seq[n * T + t - 1] > 0) ? 1.f : 0.f;
    if (m == 0.f) {
        for (int v = threadIdx.x; v < V1; v += blockDim.x) d[v] = 0.f;
        if (threadIdx.x == 0) terms[item] = terms[NT + item] = terms[2 * NT + item] = 0.f;
        return;
    }
    const float* p = lp + n * ld_lp + (long)t * V1;
    const float* q = lo + item * V1;
    float kl = 0.f, so = 0.f;
    for (int v = threadIdx.x; v < V1; v += blockDim.x) {
        const float l = q[v], e = expf(l);
        kl += e * (l - p[v]);
        so += e;
    }
    for (int o = 16; o > 0; o >>= 1) {
        kl += __shfl_xor_sync(0xffffffffu, kl, o);
        so += __shfl_xor_sync(0xffffffffu, so, o);
    }
    if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = kl; red[1][threadIdx.x >> 5] = so; }
    __syncthreads();
    kl = 0.f; so = 0.f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { kl += red[0][w]; so += red[1][w]; }
    const long long tok = seq[item];
    const float a = adv[n];
    const float ratio = expf(p[tok] - q[tok]);
    const float clamped = fminf(fmaxf(ratio, 1.f - eps), 1.f + eps);
    const float pg1 = -a * ratio, pg2 = -a * clamped;
    const bool unclamped = (ratio >= 1.f - eps && ratio <= 1.f + eps) || pg1 > pg2;
    const float g_pick = unclamped ? -a * ratio : 0.f;
    const float coef = per_row ? m : m * upstream / (*mask_sum);
    const float gsum = coef * (g_pick - kl_coef * so);
    for (int v = threadIdx.x; v < V1; v += blockDim.x) {
        const float g = coef * ((v == tok ? g_pick : 0.f) - kl_coef * expf(q[v]));
        d[v] = g - expf(p[v]) * gsum;
    }
    if (threadIdx.x == 0) {
        terms[item] = fmaxf(pg1, pg2);
        terms[NT + item] = kl;
        terms[2 * NT + item] = fabsf(ratio - 1.f) > eps ? 1.f : 0.f;
    }
}

// single CTA: the masked means (pg_loss, kl_loss, clipfrac, and loss = pg_loss + kl_coef kl_loss), each row's masked mean of
// pg + kl_coef kl (reduction 'none'), and the rewarded scores in fp32 (losses.py:302: scores.type_as(input))
__global__ void __launch_bounds__(256) ppo_reduce_kernel(const float* __restrict__ terms, const float* __restrict__ row_msum, const double* __restrict__ scores,
                                                         int N, int T, float kl_coef, float* __restrict__ row_loss, float* __restrict__ scores_out,
                                                         float* __restrict__ loss, float* __restrict__ pg_loss, float* __restrict__ kl_loss,
                                                         float* __restrict__ clipfrac) {
    __shared__ float sh[4][256];
    const long NT = (long)N * T;
    float a_pg = 0.f, a_kl = 0.f, a_cl = 0.f, a_m = 0.f;
    for (int n = threadIdx.x; n < N; n += 256) {
        float r_pg = 0.f, r_kl = 0.f, r_cl = 0.f;
        for (int t = 0; t < T; ++t) {
            const long i = (long)n * T + t;
            r_pg += terms[i]; r_kl += terms[NT + i]; r_cl += terms[2 * NT + i];
        }
        const float ms = row_msum[n];
        row_loss[n] = (r_pg + kl_coef * r_kl) / ms;
        scores_out[n] = (float)scores[n];
        a_pg += r_pg; a_kl += r_kl; a_cl += r_cl; a_m += ms;
    }
    sh[0][threadIdx.x] = a_pg; sh[1][threadIdx.x] = a_kl; sh[2][threadIdx.x] = a_cl; sh[3][threadIdx.x] = a_m;
    __syncthreads();
    for (int w = 128; w > 0; w >>= 1) {
        if (threadIdx.x < w)
            for (int k = 0; k < 4; ++k) sh[k][threadIdx.x] += sh[k][threadIdx.x + w];
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const float pg = sh[0][0] / sh[3][0], kl = sh[1][0] / sh[3][0];
        *pg_loss = pg; *kl_loss = kl; *clipfrac = sh[2][0] / sh[3][0];
        if (loss != nullptr) *loss = pg + kl_coef * kl;
    }
}

// drop_worst: row n of d logits [N, cols] times row_coef[n] (upstream / (k * row mask count) for kept rows, 0 for dropped ones)
__global__ void ppo_scale_rows_kernel(float* __restrict__ dl, long n, long cols, const float* __restrict__ row_coef) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) dl[i] *= row_coef[i / cols];
}

// nn.LSTMCell backward (gate pre-activations saved): dgates [rows, 4H] (i,f,g,o) and dc_prev from dh, dc
__global__ void lstm_cell_backward_kernel(int rows, int H, const float* __restrict__ gates, const float* __restrict__ c_prev, const float* __restrict__ c_new,
                                          const float* __restrict__ dh, const float* __restrict__ dh_extra, long ld_extra, uint32_t drop_site,
                                          uint32_t drop_step, unsigned long long seed, float p, float* __restrict__ dc_carry,
                                          float* __restrict__ dgates) {
    const long total = (long)rows * H;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int r = (int)(i / H), c = (int)(i % H);
        const float* g = gates + (long)r * 4 * H;
        const float ig = 1.f / (1.f + expf(-g[c])), fg = 1.f / (1.f + expf(-g[H + c])), gg = tanhf(g[2 * H + c]), og = 1.f / (1.f + expf(-g[3 * H + c]));
        const float cp = c_prev ? c_prev[i] : 0.f;
        const float tc = tanhf(c_new[i]);
        float dht = dh[i];
        if (dh_extra != nullptr) dht += dh_extra[(long)r * ld_extra + c] * (drop_site ? drop_scale(seed, drop_site, drop_step, (uint32_t)i, p) : 1.f);
        const float dc = dc_carry[i] + dht * og * (1.f - tc * tc);
        float* dg = dgates + (long)r * 4 * H;
        dg[c] = dc * gg * ig * (1.f - ig);
        dg[H + c] = dc * cp * fg * (1.f - fg);
        dg[2 * H + c] = dc * ig * (1.f - gg * gg);
        dg[3 * H + c] = dht * tc * og * (1.f - og);
        dc_carry[i] = dc * fg;
    }
}

// Maxout cell backward (Att2in2Core, AttModel.py:773-787; pre-activation sums saved): s [rows, 5H] = (i, f, o, a, b) with
// c' = sigmoid(f) c + sigmoid(i) max(a, b), h' = sigmoid(o) tanh(c').  d max goes to the larger of a, b; a tie splits it half-and-half,
// as torch.maximum's autograd does.  dh_extra / drop_* as in lstm_cell_backward.
__global__ void maxout_cell_backward_kernel(int rows, int H, const float* __restrict__ sums, const float* __restrict__ c_prev, const float* __restrict__ c_new,
                                            const float* __restrict__ dh, const float* __restrict__ dh_extra, long ld_extra, uint32_t drop_site,
                                            uint32_t drop_step, unsigned long long seed, float p, float* __restrict__ dc_carry, float* __restrict__ dsums) {
    const long total = (long)rows * H;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int r = (int)(i / H), c = (int)(i % H);
        const float* s = sums + (long)r * 5 * H;
        const float ig = 1.f / (1.f + expf(-s[c])), fg = 1.f / (1.f + expf(-s[H + c])), og = 1.f / (1.f + expf(-s[2 * H + c]));
        const float a = s[3 * H + c], b = s[4 * H + c];
        const float gg = fmaxf(a, b);
        const float cp = c_prev ? c_prev[i] : 0.f;
        const float tc = tanhf(c_new[i]);
        float dht = dh[i];
        if (dh_extra != nullptr) dht += dh_extra[(long)r * ld_extra + c] * (drop_site ? drop_scale(seed, drop_site, drop_step, (uint32_t)i, p) : 1.f);
        const float dc = dc_carry[i] + dht * og * (1.f - tc * tc);
        const float dg = dc * ig;
        float* ds = dsums + (long)r * 5 * H;
        ds[c] = dc * gg * ig * (1.f - ig);
        ds[H + c] = dc * cp * fg * (1.f - fg);
        ds[2 * H + c] = dht * tc * og * (1.f - og);
        ds[3 * H + c] = a > b ? dg : (a < b ? 0.f : 0.5f * dg);
        ds[4 * H + c] = b > a ? dg : (b < a ? 0.f : 0.5f * dg);
        dc_carry[i] = dc * fg;
    }
}

// Additive attention backward in two kernels (rpi rows per image):
//   in : d_out[rows,H] (grad of the attended vector), alpha[rows,R], att_h[rows,A], p_att[B,R,A], att[B,R,H], w[A]
//   out: d_att_h[rows,A] (overwritten); accumulated: d_att[B,R,H], d_p_att[B,R,A]; atomically accumulated: d_w[A], d_b[1]
// (1) d alpha[row, r] = <d_out[row], att[img, r, :]>, one warp per (row, region)
constexpr int AB_MAX_RPI = 16;
__global__ void __launch_bounds__(256) attention_dalpha_kernel(int items, int rpi, int R, int H, const float* __restrict__ d_out, const float* __restrict__ att,
                                                               float* __restrict__ d_alpha) {
    const int item = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (item >= items) return;
    const int row = item / R, r = item % R, img = row / rpi;
    const float4* dr = reinterpret_cast<const float4*>(d_out + (long)row * H);
    const float4* ar = reinterpret_cast<const float4*>(att + ((long)img * R + r) * H);
    float s = 0.f;
    for (int c = lane; c < H / 4; c += 32) {
        const float4 x = dr[c], y = ar[c];
        s = fmaf(x.x, y.x, s); s = fmaf(x.y, y.y, s); s = fmaf(x.z, y.z, s); s = fmaf(x.w, y.w, s);
    }
    for (int c = (H / 4) * 4 + lane; c < H; c += 32) s = fmaf(d_out[(long)row * H + c], att[((long)img * R + r) * H + c], s);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) d_alpha[item] = s;
}

// (2) grid (image, chunk of 32 hidden indices): softmax backward re-derived per CTA (rpi*R values), then the tanh path with the
// regions split over 8 thread groups and reduced through shared memory; the CTA also owns regions r = chunk, chunk + nchunks, ... for d_att.
__global__ void __launch_bounds__(256) attention_backward_kernel(int rpi, int R, int A, int H, const float* __restrict__ d_out, const float* __restrict__ alpha,
                                                                 const float* __restrict__ d_alpha, const float* __restrict__ att_h,
                                                                 const float* __restrict__ p_att, const float* __restrict__ w, float* __restrict__ d_att_h,
                                                                 float* __restrict__ d_att, float* __restrict__ d_p_att, float* __restrict__ d_w,
                                                                 float* __restrict__ d_b) {
    extern __shared__ float sm[];
    float* s_ds = sm;                       // [rpi][R]  d alpha, then d score
    float* s_al = s_ds + rpi * R;           // [rpi][R]  alpha
    float* s_red = s_al + rpi * R;          // [8][32][rpi + 1]
    const int img = blockIdx.x, chunk = blockIdx.y, nchunks = gridDim.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < rpi * R; i += 256) {
        s_al[i] = alpha[(long)img * rpi * R + i];
        s_ds[i] = d_alpha[(long)img * rpi * R + i];
    }
    __syncthreads();
    for (int j = warp; j < rpi; j += 8) {
        float dot = 0.f;
        for (int r = lane; r < R; r += 32) dot = fmaf(s_al[j * R + r], s_ds[j * R + r], dot);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
        float bsum = 0.f;
        for (int r = lane; r < R; r += 32) {
            const float ds = s_al[j * R + r] * (s_ds[j * R + r] - dot);
            s_ds[j * R + r] = ds;
            bsum += ds;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) bsum += __shfl_xor_sync(0xffffffffu, bsum, o);
        if (lane == 0 && chunk == 0) atomicAdd(d_b, bsum);
    }
    __syncthreads();
    // d att[img, r, c] += sum_j alpha[j, r] * d_out[j, c] for this CTA's regions
    for (int r = chunk; r < R; r += nchunks) {
        for (int c = threadIdx.x; c < H; c += 256) {
            float s = 0.f;
            for (int j = 0; j < rpi; ++j) s = fmaf(s_al[j * R + r], d_out[((long)img * rpi + j) * H + c], s);
            d_att[((long)img * R + r) * H + c] += s;
        }
    }
    // through w . tanh(p_att + att_h): lane = hidden index inside the chunk, warp = region group
    const int a = chunk * 32 + lane;
    float dw = 0.f;
    float dah[AB_MAX_RPI];
#pragma unroll
    for (int j = 0; j < AB_MAX_RPI; ++j) dah[j] = 0.f;
    if (a < A) {
        const float wa = w[a];
        float ah[AB_MAX_RPI];
#pragma unroll
        for (int j = 0; j < AB_MAX_RPI; ++j) ah[j] = j < rpi ? att_h[((long)img * rpi + j) * A + a] : 0.f;
        for (int r = warp; r < R; r += 8) {
            const float pv = p_att[((long)img * R + r) * A + a];
            float dp = 0.f;
#pragma unroll
            for (int j = 0; j < AB_MAX_RPI; ++j) {
                if (j < rpi) {
                    const float th = tanhf(pv + ah[j]);
                    const float ds = s_ds[j * R + r];
                    dw = fmaf(ds, th, dw);
                    const float dz = ds * wa * (1.f - th * th);
                    dp += dz;
                    dah[j] += dz;
                }
            }
            d_p_att[((long)img * R + r) * A + a] += dp;
        }
    }
    float* red = s_red + (warp * 32 + lane) * (rpi + 1);
#pragma unroll
    for (int j = 0; j < AB_MAX_RPI; ++j)
        if (j < rpi) red[j] = dah[j];
    red[rpi] = dw;
    __syncthreads();
    for (int i = threadIdx.x; i < 32 * (rpi + 1); i += 256) {
        const int l = i / (rpi + 1), j = i % (rpi + 1);
        float s = 0.f;
#pragma unroll
        for (int g = 0; g < 8; ++g) s += s_red[(g * 32 + l) * (rpi + 1) + j];
        const int aa = chunk * 32 + l;
        if (aa >= A) continue;
        if (j < rpi) d_att_h[((long)img * rpi + j) * A + aa] = s;
        else atomicAdd(d_w + aa, s);
    }
}

// y = dy * (x > 0 ? scale : 0): backward of Dropout(ReLU(.)) given the saved post-dropout activation x
__global__ void relu_dropout_backward_kernel(long n, const float* __restrict__ x, const float* __restrict__ dy, float* __restrict__ dx, float scale) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) dx[i] = x[i] > 0.f ? dy[i] * scale : 0.f;
}

// d_emb[tok[r], :] += d_xt[r, :] * (xt[r, :] > 0 ? scale : 0)
__global__ void embed_backward_kernel(int rows, int E, const int* __restrict__ tokens, const float* __restrict__ xt, const float* __restrict__ dxt, long ld_dxt,
                                      float scale, float* __restrict__ d_emb) {
    const int r = blockIdx.x;
    float* d = d_emb + (long)tokens[r] * E;
    for (int c = threadIdx.x; c < E; c += blockDim.x) {
        if (xt[(long)r * E + c] > 0.f) atomicAdd(d + c, dxt[(long)r * ld_dxt + c] * scale);
    }
}

// d_emb[tok[r], :] += d_xt[r, :]: backward of a bare nn.Embedding lookup (NewFC, AttModel.py:908), no ReLU gate and no dropout
__global__ void embed_scatter_kernel(int rows, int E, const int* __restrict__ tokens, const float* __restrict__ dxt, long ld_dxt, float* __restrict__ d_emb) {
    const int r = blockIdx.x;
    float* d = d_emb + (long)tokens[r] * E;
    for (int c = threadIdx.x; c < E; c += blockDim.x) atomicAdd(d + c, dxt[(long)r * ld_dxt + c]);
}

// out[img, c] (+)= sum over the image's rows and all steps of x[step][row, c]
// grid (images, column slices of 256): one column per thread, the steps x rpi terms of a column four loads at a time
// (the first version ran one CTA per image over all columns: 10 CTAs for the whole GPU, 196 us for [20 x 50 x 4096])
__global__ void per_image_sum_kernel(int steps, int rows, int rpi, int cols, const float* __restrict__ x, float* __restrict__ out) {
    const int img = blockIdx.x;
    const int c = blockIdx.y * blockDim.x + threadIdx.x;
    if (c >= cols) return;
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
    const int n = steps * rpi;
    int i = 0;
    auto at = [&](int k) { return x[((long)(k / rpi) * rows + (long)img * rpi + (k % rpi)) * cols + c]; };
    for (; i + 4 <= n; i += 4) { s0 += at(i); s1 += at(i + 1); s2 += at(i + 2); s3 += at(i + 3); }
    for (; i < n; ++i) s0 += at(i);
    out[(long)img * cols + c] = (s0 + s1) + (s2 + s3);
}

__global__ void add_strided_kernel(float* a, const float* b, long ld_b, int rows, int cols) {
    const long n = (long)rows * cols;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) a[i] += b[(i / cols) * ld_b + (i % cols)];
}

int nblocks(long n) {
    long b = (n + 255) / 256;
    return (int)(b > sm_count() * 8 ? sm_count() * 8 : (b < 1 ? 1 : b));
}

}  // namespace

#define LAUNCH_OK()                         \
    CAPB_CHECK_CUDA(cudaGetLastError());    \
    return 0

int dropout_apply_launch(float* x, int rows, int cols, long ld, unsigned long long seed, unsigned site, unsigned step, float p, cudaStream_t st) {
    if (p <= 0.f || rows <= 0) return 0;
    dropout_apply_kernel<<<nblocks((long)rows * cols), 256, 0, st>>>(x, (long)rows * cols, cols, ld, seed, site, step, p);
    LAUNCH_OK();
}
int dropout_mask_launch(float* m, long n, unsigned long long seed, unsigned site, unsigned step, float p, cudaStream_t st) {
    dropout_mask_kernel<<<nblocks(n), 256, 0, st>>>(m, n, seed, site, step, p);
    LAUNCH_OK();
}
int dropout_copy_launch(const float* x, long ld_x, float* y, long ld_y, int rows, int cols, unsigned long long seed, unsigned site, unsigned step, float p,
                        cudaStream_t st) {
    dropout_copy_kernel<<<nblocks((long)rows * cols), 256, 0, st>>>(x, ld_x, y, ld_y, rows, cols, seed, site, step, p);
    LAUNCH_OK();
}
int embed_relu_dropout_launch(int rows, int E, const int* tokens, const float* emb, float* xt, unsigned long long seed, unsigned step, float p,
                              cudaStream_t st) {
    embed_relu_dropout_kernel<<<rows, 128, 0, st>>>(rows, E, tokens, emb, xt, seed, step, p);
    LAUNCH_OK();
}
int scst_dlogits_launch(const float* logp, long ld_row, const long long* seq, const float* reward, const float* mask_sum, float upstream, int N, int T, int V1,
                        float* dl, cudaStream_t st, const float* row_coef) {
    scst_dlogits_kernel<<<N * T, 256, 0, st>>>(logp, ld_row, seq, reward, mask_sum, upstream, T, V1, dl, row_coef);
    LAUNCH_OK();
}
int scst_drop_worst_launch(const long long* seq, const float* row_loss, int N, int T, int keep, float upstream, float* row_msum, float* row_coef, float* loss,
                           cudaStream_t st) {
    CAPB_REQUIRE(keep >= 1 && keep <= N, "drop_worst: the number of kept rows must be in 1..rows");
    scst_row_mask_kernel<<<cdiv(N, 128), 128, 0, st>>>(seq, N, T, row_msum);
    CAPB_CHECK_CUDA(cudaGetLastError());
    drop_worst_select_kernel<<<1, 256, 0, st>>>(row_loss, row_msum, N, keep, upstream, row_coef, loss);
    LAUNCH_OK();
}
int xe_loss_backward_launch(const float* logp, long ld_row, const long long* labels, long ld_l, const float* masks, long ld_m, int N, int steps, int Ls, int V1,
                            float smoothing, float upstream, float* mask_sum, float* item_loss, float* dl, float* loss, cudaStream_t st, int keep,
                            float* row_loss, float* row_msum, float* row_coef) {
    xe_mask_sum_kernel<<<1, 256, 0, st>>>(masks, ld_m, N, Ls, mask_sum);
    CAPB_CHECK_CUDA(cudaGetLastError());
    xe_dlogits_kernel<<<N * steps, 256, 0, st>>>(logp, ld_row, labels, ld_l, masks, ld_m, mask_sum, upstream, smoothing, steps, V1, dl, item_loss, nullptr);
    CAPB_CHECK_CUDA(cudaGetLastError());
    if (keep > 0) {      // drop_worst: per-row losses, selection, then the gradient pass again with the per-row coefficients
        CAPB_REQUIRE(keep <= N && row_loss && row_msum && row_coef, "drop_worst: bad arguments");
        xe_row_loss_kernel<<<cdiv(N, 128), 128, 0, st>>>(item_loss, N, steps, Ls, masks, ld_m, smoothing, V1, row_loss, row_msum);
        CAPB_CHECK_CUDA(cudaGetLastError());
        drop_worst_select_kernel<<<1, 256, 0, st>>>(row_loss, row_msum, N, keep, upstream, row_coef, loss);
        CAPB_CHECK_CUDA(cudaGetLastError());
        xe_dlogits_kernel<<<N * steps, 256, 0, st>>>(logp, ld_row, labels, ld_l, masks, ld_m, mask_sum, upstream, smoothing, steps, V1, dl, item_loss, row_coef);
        LAUNCH_OK();
    }
    xe_loss_kernel<<<1, 256, 0, st>>>(item_loss, N, steps, Ls, masks, ld_m, smoothing, V1, mask_sum, loss);
    LAUNCH_OK();
}
int ppo_shift_launch(const long long* seq, int N, int T, long long* tokens_in, cudaStream_t st) {
    ppo_shift_kernel<<<cdiv(N * T, 256), 256, 0, st>>>(seq, N, T, tokens_in);
    LAUNCH_OK();
}
int ppo_loss_backward_launch(const float* lp, long ld_lp, const float* lo, const long long* seq, const float* adv, const double* scores, int N, int T, int V1,
                             float cliprange, float kl_coef, float upstream, int keep, const PpoScratch& s, float* dl, float* scores_out, float* loss,
                             float* row_loss, float* pg_loss, float* kl_loss, float* clipfrac, cudaStream_t st) {
    CAPB_REQUIRE(keep >= 0 && keep <= N, "drop_worst: the number of kept rows must be in 0..rows");
    ppo_mask_kernel<<<1, 256, 0, st>>>(seq, N, T, s.row_msum, s.mask_sum);
    CAPB_CHECK_CUDA(cudaGetLastError());
    ppo_row_kernel<<<N * T, 256, 0, st>>>(lp, ld_lp, lo, seq, adv, s.mask_sum, upstream, keep > 0, cliprange, kl_coef, T, V1, dl, s.terms);
    CAPB_CHECK_CUDA(cudaGetLastError());
    ppo_reduce_kernel<<<1, 256, 0, st>>>(s.terms, s.row_msum, scores, N, T, kl_coef, row_loss, scores_out, keep > 0 ? nullptr : loss, pg_loss, kl_loss, clipfrac);
    CAPB_CHECK_CUDA(cudaGetLastError());
    if (keep > 0) {
        drop_worst_select_kernel<<<1, 256, 0, st>>>(row_loss, s.row_msum, N, keep, upstream, s.row_coef, loss);
        CAPB_CHECK_CUDA(cudaGetLastError());
        const long cols = (long)T * V1;
        ppo_scale_rows_kernel<<<nblocks(N * cols), 256, 0, st>>>(dl, N * cols, cols, s.row_coef);
    }
    LAUNCH_OK();
}
int logsoftmax_vjp_launch(const float* logp, const float* g, long ld_row, const long long* seq, int N, int T, int V1, float* dl, cudaStream_t st) {
    const bool vec = V1 % 4 == 0 && ld_row % 4 == 0 && (reinterpret_cast<uintptr_t>(logp) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(dl)) % 16 == 0;
    if (vec) logsoftmax_vjp_kernel<4><<<N * T, 256, 0, st>>>(logp, g, ld_row, seq, T, V1, dl);
    else logsoftmax_vjp_kernel<1><<<N * T, 256, 0, st>>>(logp, g, ld_row, seq, T, V1, dl);
    LAUNCH_OK();
}
int lstm_cell_backward_launch(int rows, int H, const float* gates, const float* c_prev, const float* c_new, const float* dh, const float* dh_extra,
                              long ld_extra, unsigned drop_site, unsigned drop_step, unsigned long long seed, float p, float* dc_carry, float* dgates,
                              cudaStream_t st) {
    lstm_cell_backward_kernel<<<nblocks((long)rows * H), 256, 0, st>>>(rows, H, gates, c_prev, c_new, dh, dh_extra, ld_extra, drop_site, drop_step, seed, p,
                                                                        dc_carry, dgates);
    LAUNCH_OK();
}
int maxout_cell_backward_launch(int rows, int H, const float* sums, const float* c_prev, const float* c_new, const float* dh, const float* dh_extra,
                                long ld_extra, unsigned drop_site, unsigned drop_step, unsigned long long seed, float p, float* dc_carry, float* dsums,
                                cudaStream_t st) {
    maxout_cell_backward_kernel<<<nblocks((long)rows * H), 256, 0, st>>>(rows, H, sums, c_prev, c_new, dh, dh_extra, ld_extra, drop_site, drop_step, seed, p,
                                                                          dc_carry, dsums);
    LAUNCH_OK();
}
int attention_backward_launch(int n_images, int rpi, int R, int A, int H, const float* d_out, const float* alpha, const float* att_h, const float* p_att,
                              const float* att, const float* w, float* d_att_h, float* d_att, float* d_p_att, float* d_w, float* d_b, float* d_alpha_scratch,
                              cudaStream_t st) {
    CAPB_REQUIRE(rpi <= AB_MAX_RPI, "attention backward handles up to 16 rows per image");
    CAPB_REQUIRE(H % 4 == 0, "attention backward needs rnn_size % 4 == 0");
    const int items = n_images * rpi * R;
    attention_dalpha_kernel<<<cdiv(items, 8), 256, 0, st>>>(items, rpi, R, H, d_out, att, d_alpha_scratch);
    CAPB_CHECK_CUDA(cudaGetLastError());
    const size_t smem = sizeof(float) * (2 * (size_t)rpi * R + 256 * (rpi + 1));
    // d alpha and alpha of the image's rows are staged whole: past the default 48 KB above about 248 regions at 16 rows per image
    // (148 KB at 1024 regions)
    CAPB_REQUIRE(smem <= 200 * 1024, "attention backward: rows per image x regions too large for the shared-memory staging");
    static std::atomic<unsigned long long> configured{0};
    if (first_use_on_device(configured)) {
        CAPB_CHECK_CUDA(cudaFuncSetAttribute(attention_backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    }
    attention_backward_kernel<<<dim3(n_images, cdiv(A, 32)), 256, smem, st>>>(rpi, R, A, H, d_out, alpha, d_alpha_scratch, att_h, p_att, w, d_att_h, d_att, d_p_att,
                                                                             d_w, d_b);
    LAUNCH_OK();
}
int relu_dropout_backward_launch(long n, const float* x, const float* dy, float* dx, float scale, cudaStream_t st) {
    relu_dropout_backward_kernel<<<nblocks(n), 256, 0, st>>>(n, x, dy, dx, scale);
    LAUNCH_OK();
}
int embed_backward_launch(int rows, int E, const int* tokens, const float* xt, const float* dxt, long ld_dxt, float scale, float* d_emb, cudaStream_t st) {
    embed_backward_kernel<<<rows, 128, 0, st>>>(rows, E, tokens, xt, dxt, ld_dxt, scale, d_emb);
    LAUNCH_OK();
}
int embed_scatter_launch(int rows, int E, const int* tokens, const float* dxt, long ld_dxt, float* d_emb, cudaStream_t st) {
    embed_scatter_kernel<<<rows, 128, 0, st>>>(rows, E, tokens, dxt, ld_dxt, d_emb);
    LAUNCH_OK();
}
int per_image_sum_launch(int steps, int rows, int rpi, int cols, const float* x, float* out, cudaStream_t st) {
    per_image_sum_kernel<<<dim3(rows / rpi, cdiv(cols, 256)), 256, 0, st>>>(steps, rows, rpi, cols, x, out);
    LAUNCH_OK();
}
int add_strided_launch(float* a, const float* b, long ld_b, int rows, int cols, cudaStream_t st) {
    add_strided_kernel<<<nblocks((long)rows * cols), 256, 0, st>>>(a, b, ld_b, rows, cols);
    LAUNCH_OK();
}

CAPB_DEFINE_SALT_SETTER(dropout_salt_set_scst)

}  // namespace capb200
