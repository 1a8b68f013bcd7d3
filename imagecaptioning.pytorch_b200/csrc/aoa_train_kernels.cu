// Training-only kernels of the AoANet SCST step (forward variants with replayable dropout, and the backward passes):
//   layer_norm backward          captioning/models/TransformerModel.py:76-87   (a*(x-mean)/(std_unbiased+eps)+b)
//   GLU backward                 nn.GLU, AoAModel.py:41,143
//   refiner self-attention       AoAModel.py:56-98 with TransformerModel.attention (:152-162), dropout on the probabilities
//   decoder multi-head attention AoAModel.py:168 (single query per row over the image's K | V halves of ctx2att's output)
//   mean-pool backward           AoAModel.py:214-216
#include "common.cuh"
#include "dropout.cuh"
#include "kernels.cuh"
#include "attn.cuh"

namespace capb200 {

namespace {

__device__ __forceinline__ float wsum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float wmax(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// one CTA of 128 threads per row: dx (+)= d LayerNorm / dx; stats[row] = (mean, 1/(std+eps)) for the parameter-gradient pass
__device__ __forceinline__ float bsum128(float v, float* sh) {
    v = wsum(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    return (sh[0] + sh[1]) + (sh[2] + sh[3]);
}
// add1 / add2 (optional): two more addends of the output row (the other branches that reach the LayerNorm input), folded in here instead
// of separate copy / add launches:  dx = [dx +] add1 + add2 + dLN
__global__ void __launch_bounds__(128) ln_backward_kernel(int rows, int D, const float* __restrict__ x, long ld_x, const float* __restrict__ a,
                                                          const float* __restrict__ dy, long ld_dy, float eps, float* __restrict__ dx, long ld_dx,
                                                          int accumulate, float2* __restrict__ stats, const float* __restrict__ add1, long ld_a1,
                                                          const float* __restrict__ add2, long ld_a2) {
    __shared__ float sh[4];
    const int row = blockIdx.x;
    const float* xr = x + (long)row * ld_x;
    const float* gr = dy + (long)row * ld_dy;
    float s = 0.f;
    for (int c = threadIdx.x; c < D; c += 128) s += xr[c];
    const float mean = bsum128(s, sh) / (float)D;
    float q = 0.f;
    for (int c = threadIdx.x; c < D; c += 128) { const float d = xr[c] - mean; q = fmaf(d, d, q); }
    const float stdv = sqrtf(bsum128(q, sh) / (float)(D - 1));
    const float inv = 1.0f / (stdv + eps);
    float g_sum = 0.f, g_dot = 0.f;                  // sum of g and of g * (x - mean), g = dy * a
    for (int c = threadIdx.x; c < D; c += 128) {
        const float g = gr[c] * __ldg(a + c);
        g_sum += g;
        g_dot = fmaf(g, xr[c] - mean, g_dot);
    }
    g_sum = bsum128(g_sum, sh);
    g_dot = bsum128(g_dot, sh);
    const float g_mean = g_sum / (float)D;
    const float k = (stdv > 0.f) ? inv * inv * g_dot / ((float)(D - 1) * stdv) : 0.f;
    for (int c = threadIdx.x; c < D; c += 128) {
        float v = inv * (gr[c] * __ldg(a + c) - g_mean) - k * (xr[c] - mean);
        if (add1 != nullptr) v += add1[(long)row * ld_a1 + c];
        if (add2 != nullptr) v += add2[(long)row * ld_a2 + c];
        float* o = dx + (long)row * ld_dx + c;
        *o = accumulate ? *o + v : v;
    }
    if (threadIdx.x == 0 && stats != nullptr) stats[row] = make_float2(mean, inv);
}

// thread per column: da[c] (+)= sum_rows dy * xhat, db[c] (+)= sum_rows dy
__global__ void ln_param_grad_kernel(int rows, int D, const float* __restrict__ x, long ld_x, const float* __restrict__ dy, long ld_dy,
                                     const float2* __restrict__ stats, float* __restrict__ da, float* __restrict__ db, int accumulate) {
    // block = 32 columns x 8 row groups (see colsum_kernel): coalesced row segments, eight independent partial sums per column
    __shared__ float sha[8][33], shb[8][33];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + tx;
    float sa = 0.f, sb = 0.f;
    if (c < D) {
        for (int r = ty; r < rows; r += 8) {
            const float2 st = stats[r];
            const float g = dy[(long)r * ld_dy + c];
            sa = fmaf(g, (x[(long)r * ld_x + c] - st.x) * st.y, sa);
            sb += g;
        }
    }
    sha[ty][tx] = sa;
    shb[ty][tx] = sb;
    __syncthreads();
    if (ty == 0 && c < D) {
        float ta = 0.f, tb = 0.f;
#pragma unroll
        for (int g = 0; g < 8; ++g) { ta += sha[g][tx]; tb += shb[g][tx]; }
        da[c] = accumulate ? da[c] + ta : ta;
        db[c] = accumulate ? db[c] + tb : tb;
    }
}

// y = t[:, :H] * sigmoid(t[:, H:]):  dt[:, :H] = dy * s,  dt[:, H:] = dy * t[:, :H] * s * (1 - s)
__global__ void glu_backward_kernel(int rows, int H, const float* __restrict__ t, long ld_t, const float* __restrict__ dy, long ld_dy, float* __restrict__ dt,
                                    long ld_dt) {
    const long total = (long)rows * H;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int r = (int)(i / H), j = (int)(i % H);
        const float a = t[(long)r * ld_t + j], b = t[(long)r * ld_t + H + j];
        const float s = 1.0f / (1.0f + expf(-b));
        const float g = dy[(long)r * ld_dy + j];
        dt[(long)r * ld_dt + j] = g * s;
        dt[(long)r * ld_dt + H + j] = g * a * s * (1.f - s);
    }
}

// ---- fused element-wise steps of the AoANet decoder loop (each replaces two to four launches of ~2 us + a launch boundary) --------------------
// inputs of step t, one CTA per row:  tok_dst[r] = tok_src[r];  xt[r] = dropout_2(relu(embed[tok]));  x1c[r] = mean[img] + dropout_4(out_prev[r])
__global__ void __launch_bounds__(256) aoa_step_inputs_kernel(int E, int H, int rpi, const int* __restrict__ tok_src, int* __restrict__ tok_dst,
                                                              const float* __restrict__ emb, float* __restrict__ xt, const float* __restrict__ mean, long ld_mean,
                                                              const float* __restrict__ out_prev, float* __restrict__ x1c, unsigned long long seed,
                                                              uint32_t step, float p_lm, float p_ctx) {
    const int r = blockIdx.x;
    const int tok = tok_src[r];
    if (tok_dst != nullptr && threadIdx.x == 0) tok_dst[r] = tok;
    const float* e = emb + (long)tok * E;
    for (int c = threadIdx.x; c < E; c += 256) xt[(long)r * E + c] = fmaxf(__ldg(e + c), 0.f) * drop_scale(seed, 2u, step, (uint32_t)(r * E + c), p_lm);
    const float* m = mean + (long)(r / rpi) * ld_mean;
    for (int c = threadIdx.x; c < H; c += 256) {
        float v = m[c];
        if (out_prev != nullptr) v += out_prev[(long)r * H + c] * drop_scale(seed, 4u, step, (uint32_t)(r * H + c), p_ctx);
        x1c[(long)r * H + c] = v;
    }
}

// out[r, j] = t[r, j] * sigmoid(t[r, H + j]);  outd[r, j] = dropout_3(out[r, j])        (GLU + the output dropout, AoAModel.py:143,181)
__global__ void glu_dropout_kernel(int rows, int H, const float* __restrict__ t, long ld_t, float* __restrict__ out, long ld_o, float* __restrict__ outd, long ld_d,
                                   unsigned long long seed, uint32_t step, float p) {
    const long total = (long)rows * H;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int r = (int)(i / H), j = (int)(i % H);
        const float a = t[(long)r * ld_t + j], b = t[(long)r * ld_t + H + j];
        const float v = a * (1.0f / (1.0f + expf(-b)));
        out[(long)r * ld_o + j] = v;
        outd[(long)r * ld_d + j] = v * drop_scale(seed, 3u, step, (uint32_t)i, p);
    }
}

// d out = dropout_3(d outd) + d ctx (what step t+1 received through its context input);  then the GLU backward of glu_backward_kernel
__global__ void glu_backward_fused_kernel(int rows, int H, const float* __restrict__ t, long ld_t, const float* __restrict__ d_outd, long ld_dd,
                                          const float* __restrict__ dctx, float* __restrict__ dt, long ld_dt, unsigned long long seed, uint32_t step, float p) {
    const long total = (long)rows * H;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int r = (int)(i / H), j = (int)(i % H);
        const float g = d_outd[(long)r * ld_dd + j] * drop_scale(seed, 3u, step, (uint32_t)i, p) + dctx[i];
        const float a = t[(long)r * ld_t + j], b = t[(long)r * ld_t + H + j];
        const float sg = 1.0f / (1.0f + expf(-b));
        dt[(long)r * ld_dt + j] = g * sg;
        dt[(long)r * ld_dt + H + j] = g * a * sg * (1.f - sg);
    }
}

// ---- sequence self-attention, train mode (dropout on the probabilities) --------------------------------------------------------------
// Shared by the AoANet refiner / Transformer encoder (all regions attend to all regions, rows image-major) and the Transformer decoder
// (causal, rows TIME-major so that the same buffers serve the step-by-step sampling pass and the batched teacher-forced pass).
//   row(b, pos) = b * b_stride + pos * p_stride;  q, k, v: [rows, ld] with the head at columns [head*dk, (head+1)*dk)
//   queries [q_lo, q_hi) of every sequence; keys [0, n_keys) (causal: key r is visible to query qi iff r <= qi)
//   key_mask [b, ld_mask] (0 = masked) or nullptr;  dropout element index = ((b*heads + head)*idx_L + qi)*idx_L + r
// Grid (sequences, heads, query chunks): the chunks split the query range (forward) or the output elements (backward) so that a
// 10-image batch still fills the machine (80 CTAs, one per (sequence, head), leave most SMs idle and make every launch long).
struct SeqAttn {
    int n_keys, dk, heads, q_lo, q_hi, causal, idx_L;
    long b_stride, p_stride, ld;
    float scale, p_drop;
    unsigned long long seed;
    uint32_t site;
    const float* key_mask;
    long ld_mask;
};

// Shared-memory rows are padded to W = dk + 4 floats: rows stay 16-byte aligned, so every inner product walks them with 128-bit loads
// (one LDS.128 per four multiply-adds instead of two or three LDS.32 per multiply-add; the scalar form was shared-memory-bandwidth
// bound: 72 us per backward launch at 36 regions x 128 columns), and W/4 = 33 chunks per row keeps the per-lane row starts on distinct banks.
__device__ __forceinline__ float dot4(const float4& a, const float4& b, float s) { return fmaf(a.x, b.x, fmaf(a.y, b.y, fmaf(a.z, b.z, fmaf(a.w, b.w, s)))); }

__global__ void __launch_bounds__(256) seq_attn_train_kernel(SeqAttn a, const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v,
                                                             float* __restrict__ out, long ld_out) {
    extern __shared__ __align__(16) float sm[];
    const int R = a.n_keys, dk = a.dk, W = dk + 4, dk4 = dk >> 2;
    float* sk = sm;                 // [R][W]
    float* sv = sk + R * W;
    float* sq = sv + R * W;         // [warps][dk]
    float* sp = sq + 8 * dk;        // [warps][R]
    const int b = blockIdx.x, head = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    const int nq = a.q_hi - a.q_lo;
    const int c_lo = a.q_lo + (int)(((long)nq * blockIdx.z) / gridDim.z), c_hi = a.q_lo + (int)(((long)nq * (blockIdx.z + 1)) / gridDim.z);
    if (c_lo >= c_hi) return;
    const int need = a.causal ? (c_hi < R ? c_hi : R) : R;      // keys this chunk can see
#pragma unroll 4
    for (int i = threadIdx.x; i < need * dk; i += blockDim.x) {       // independent coalesced loads, four in flight per thread
        const int r = i / dk, c = i % dk;
        const long g = ((long)b * a.b_stride + (long)r * a.p_stride) * a.ld + head * dk + c;
        sk[r * W + c] = k[g];
        sv[r * W + c] = v[g];
    }
    __syncthreads();
    float* p = sp + warp * R;
    float* qs = sq + warp * dk;
    for (int qi = c_lo + warp; qi < c_hi; qi += nw) {
        const long qrow = (long)b * a.b_stride + (long)qi * a.p_stride;
        for (int c = lane; c < dk; c += 32) qs[c] = q[qrow * a.ld + head * dk + c];
        __syncwarp();
        const int vis = a.causal ? (qi + 1 < need ? qi + 1 : need) : need;
        float mx = -INFINITY;
        for (int r = lane; r < vis; r += 32) {
            float s = 0.f;
            const float4* kr = reinterpret_cast<const float4*>(sk + r * W);
            const float4* q4 = reinterpret_cast<const float4*>(qs);
            for (int c = 0; c < dk4; ++c) s = dot4(q4[c], kr[c], s);
            s *= a.scale;
            if (a.key_mask != nullptr && a.key_mask[(long)b * a.ld_mask + r] == 0.f) s = -INFINITY;     // scores.masked_fill(mask == 0, -inf)  (TransformerModel.py:157-158)
            p[r] = s;
            mx = fmaxf(mx, s);
        }
        mx = wmax(mx);
        float sum = 0.f;
        for (int r = lane; r < vis; r += 32) { const float e = expf(p[r] - mx); p[r] = e; sum += e; }
        sum = wsum(sum);
        const float inv = 1.0f / sum;
        for (int r = lane; r < vis; r += 32)
            p[r] = p[r] * inv * drop_scale(a.seed, a.site, 0u, (uint32_t)((((long)b * a.heads + head) * a.idx_L + qi) * a.idx_L + r), a.p_drop);
        __syncwarp();
        for (int c4 = lane; c4 < dk4; c4 += 32) {
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int r = 0; r < vis; ++r) {
                const float w = p[r];
                const float4 x = *reinterpret_cast<const float4*>(sv + r * W + 4 * c4);
                acc.x = fmaf(w, x.x, acc.x); acc.y = fmaf(w, x.y, acc.y); acc.z = fmaf(w, x.z, acc.z); acc.w = fmaf(w, x.w, acc.w);
            }
            float* o = out + qrow * ld_out + head * dk + 4 * c4;
            o[0] = acc.x; o[1] = acc.y; o[2] = acc.z; o[3] = acc.w;
        }
        __syncwarp();
    }
}

// backward over ALL queries [0, n_keys) of a sequence: recomputes the probabilities; every chunk CTA rebuilds P and dS and writes its share
// of the dq | dk | dv elements of this (sequence, head) slice
__global__ void __launch_bounds__(256) seq_attn_backward_kernel(SeqAttn a, const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v,
                                                                const float* __restrict__ d_out, long ld_do, float* __restrict__ dq, float* __restrict__ dk_,
                                                                float* __restrict__ dv, long ld_d) {
    extern __shared__ __align__(16) float sm[];
    const int R = a.n_keys, dk = a.dk, W = dk + 4, dk4 = dk >> 2;
    float* sq = sm;                 // [R][W]
    float* sk = sq + R * W;
    float* sv = sk + R * W;
    float* sd = sv + R * W;         // d_out
    float* P = sd + R * W;          // [R][R] softmax probabilities
    float* DS = P + R * R;          // [R][R] dropout scale, then d score
    const int b = blockIdx.x, head = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
#pragma unroll 2
    for (int i = threadIdx.x; i < R * dk; i += blockDim.x) {
        const int r = i / dk, c = i % dk;
        const long row = (long)b * a.b_stride + (long)r * a.p_stride;
        const long g = row * a.ld + head * dk + c;
        sq[r * W + c] = q[g]; sk[r * W + c] = k[g]; sv[r * W + c] = v[g];
        sd[r * W + c] = d_out[row * ld_do + head * dk + c];
    }
    __syncthreads();
    // P = softmax(q k^T * scale) row by row (one warp per query row); invisible keys get probability 0
    for (int qi = warp; qi < R; qi += nw) {
        const int vis = a.causal ? qi + 1 : R;
        const float4* q4 = reinterpret_cast<const float4*>(sq + qi * W);
        float mx = -INFINITY;
        for (int r = lane; r < R; r += 32) {
            float s = -INFINITY;
            if (r < vis) {
                s = 0.f;
                const float4* kr = reinterpret_cast<const float4*>(sk + r * W);
                for (int c = 0; c < dk4; ++c) s = dot4(q4[c], kr[c], s);
                s *= a.scale;
                if (a.key_mask != nullptr && a.key_mask[(long)b * a.ld_mask + r] == 0.f) s = -INFINITY;
            }
            P[qi * R + r] = s;
            mx = fmaxf(mx, s);
        }
        mx = wmax(mx);
        float sum = 0.f;
        for (int r = lane; r < R; r += 32) { const float e = expf(P[qi * R + r] - mx); P[qi * R + r] = e; sum += e; }
        sum = wsum(sum);
        const float inv = 1.0f / sum;
        for (int r = lane; r < R; r += 32) {
            P[qi * R + r] *= inv;
            DS[qi * R + r] = drop_scale(a.seed, a.site, 0u, (uint32_t)((((long)b * a.heads + head) * a.idx_L + qi) * a.idx_L + r), a.p_drop);
        }
    }
    __syncthreads();
    const int total = R * dk4;          // output elements in units of four columns
    const int e_lo = (int)(((long)total * blockIdx.z) / gridDim.z), e_hi = (int)(((long)total * (blockIdx.z + 1)) / gridDim.z);
    // dV[r, c..c+3] = sum_qi P[qi, r] * D[qi, r] * dO[qi, c..c+3]
    for (int i = e_lo + threadIdx.x; i < e_hi; i += blockDim.x) {
        const int r = i / dk4, c = 4 * (i % dk4);
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int qi = a.causal ? r : 0; qi < R; ++qi) {
            const float w = P[qi * R + r] * DS[qi * R + r];
            const float4 x = *reinterpret_cast<const float4*>(sd + qi * W + c);
            acc.x = fmaf(w, x.x, acc.x); acc.y = fmaf(w, x.y, acc.y); acc.z = fmaf(w, x.z, acc.z); acc.w = fmaf(w, x.w, acc.w);
        }
        float* o = dv + ((long)b * a.b_stride + (long)r * a.p_stride) * ld_d + head * dk + c;
        o[0] = acc.x; o[1] = acc.y; o[2] = acc.z; o[3] = acc.w;
    }
    __syncthreads();
    // d score: dP = (dO V^T) * D ; dS = P * (dP - sum_r P dP)
    for (int qi = warp; qi < R; qi += nw) {
        const int vis = a.causal ? qi + 1 : R;
        const float4* d4 = reinterpret_cast<const float4*>(sd + qi * W);
        float dot = 0.f;
        for (int r = lane; r < R; r += 32) {
            float dp = 0.f;
            if (r < vis) {
                float s = 0.f;
                const float4* vr = reinterpret_cast<const float4*>(sv + r * W);
                for (int c = 0; c < dk4; ++c) s = dot4(d4[c], vr[c], s);
                dp = s * DS[qi * R + r];
            }
            DS[qi * R + r] = dp;
            dot = fmaf(P[qi * R + r], dp, dot);
        }
        dot = wsum(dot);
        __syncwarp();
        for (int r = lane; r < R; r += 32) DS[qi * R + r] = P[qi * R + r] * (DS[qi * R + r] - dot) * a.scale;
    }
    __syncthreads();
    for (int i = e_lo + threadIdx.x; i < e_hi; i += blockDim.x) {
        const int r = i / dk4, c = 4 * (i % dk4);
        float4 aq = make_float4(0.f, 0.f, 0.f, 0.f), ak = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int j = 0; j < R; ++j) {
            const float w1 = DS[r * R + j], w2 = DS[j * R + r];
            const float4 kk = *reinterpret_cast<const float4*>(sk + j * W + c);          // dQ[r] = sum_j dS[r, j] K[j]
            const float4 qq = *reinterpret_cast<const float4*>(sq + j * W + c);          // dK[r] = sum_j dS[j, r] Q[j]
            aq.x = fmaf(w1, kk.x, aq.x); aq.y = fmaf(w1, kk.y, aq.y); aq.z = fmaf(w1, kk.z, aq.z); aq.w = fmaf(w1, kk.w, aq.w);
            ak.x = fmaf(w2, qq.x, ak.x); ak.y = fmaf(w2, qq.y, ak.y); ak.z = fmaf(w2, qq.z, ak.z); ak.w = fmaf(w2, qq.w, ak.w);
        }
        const long g = ((long)b * a.b_stride + (long)r * a.p_stride) * ld_d + head * dk + c;
        dq[g] = aq.x; dq[g + 1] = aq.y; dq[g + 2] = aq.z; dq[g + 3] = aq.w;
        dk_[g] = ak.x; dk_[g + 1] = ak.y; dk_[g + 2] = ak.z; dk_[g + 3] = ak.w;
    }
}

// ---- decoder attention, train mode: one CTA per (row, head) (attn.cuh); probabilities (before dropout) are saved for the backward ------------
__global__ void __launch_bounds__(128) cross_attn_train_kernel(int rows, int rpi, int heads, int dk, int R, const float* __restrict__ q, long ld_q,
                                                               const float* __restrict__ kk, const float* __restrict__ vv, long ld_kv, float scale,
                                                               unsigned long long seed, uint32_t site, uint32_t step, float p_drop,
                                                               float* __restrict__ out, long ld_out, float* __restrict__ probs,
                                                               const float* __restrict__ mask, long ld_mask, int row_mod) {
    // rows may be TIME-major blocks of row_mod rows each (Transformer training: row = t * row_mod + n): the image is (row % row_mod) / rpi and the
    // dropout stream is keyed by (step + t, n), so a batched call over all t and a step-by-step sequence of calls draw the same masks
    extern __shared__ float sm[];       // [R] scores -> exp -> dropped probabilities
    __shared__ float sh_inv;
    const int item = blockIdx.x;
    const int row = item / heads, head = item % heads;
    const int local = row % row_mod;
    const uint32_t tstep = step + (uint32_t)(row / row_mod);
    const int img = local / rpi;
    const long item_local = (long)local * heads + head;
    const float* qr = q + (long)row * ld_q + head * dk;
    const float* kb = kk + (long)img * R * ld_kv + head * dk;
    const float* vb = vv + (long)img * R * ld_kv + head * dk;
    sq_attention_scores(qr, kb, ld_kv, R, dk, scale, mask != nullptr ? mask + (long)img * ld_mask : nullptr, sm);
    const float inv = sq_attention_softmax(sm, R, &sh_inv);
    for (int r = threadIdx.x; r < R; r += 128) {
        const float pr = sm[r] * inv;
        probs[(long)item * R + r] = pr;
        sm[r] = pr * drop_scale(seed, site, tstep, (uint32_t)(item_local * R + r), p_drop);
    }
    __syncthreads();
    for (int c = threadIdx.x; c < dk; c += 128) out[(long)row * ld_out + head * dk + c] = sq_attention_column(sm, vb, ld_kv, R, c);
}

// backward: one CTA per (image, head) walks the image's rpi rows; dq written, dK / dV accumulated (+=) into the per-image buffers
__global__ void __launch_bounds__(512) cross_attn_backward_kernel(int rpi, int heads, int dk, int R, const float* __restrict__ q, long ld_q,
                                                                  const float* __restrict__ kk, const float* __restrict__ vv, long ld_kv, float scale,
                                                                  unsigned long long seed, uint32_t site, uint32_t step, float p_drop,
                                                                  const float* __restrict__ probs, const float* __restrict__ d_out, long ld_do,
                                                                  float* __restrict__ dq, long ld_dq, float* __restrict__ dkk, float* __restrict__ dvv,
                                                                  long ld_dkv, int rpi1, int row_mod) {
    // rpi = rows of this image in the launch = n_steps * rpi1 (rpi1 rows per image per time block; time blocks are row_mod rows apart)
    extern __shared__ float sm[];
    const int W = dk + 1;
    float* sk = sm;                  // [R][W]
    float* sv = sk + R * W;
    float* sq = sv + R * W;          // [rpi][W]
    float* sd = sq + rpi * W;        // [rpi][W]  d_out
    float* PD = sd + rpi * W;        // [rpi][R]  p * D
    float* DS = PD + rpi * R;        // [rpi][R]  d score (scaled)
    const int img = blockIdx.x, head = blockIdx.y;
    auto row_of = [&](int j) -> long { return (long)(j / rpi1) * row_mod + (long)img * rpi1 + (j % rpi1); };
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
#pragma unroll 4
    for (int i = threadIdx.x; i < R * dk; i += blockDim.x) {       // independent coalesced loads, several in flight per thread
        const int r = i / dk, c = i % dk;
        sk[r * W + c] = kk[((long)img * R + r) * ld_kv + head * dk + c];
        sv[r * W + c] = vv[((long)img * R + r) * ld_kv + head * dk + c];
    }
    for (int i = threadIdx.x; i < rpi * dk; i += blockDim.x) {
        const int j = i / dk, c = i % dk;
        const long row = row_of(j);
        sq[j * W + c] = q[row * ld_q + head * dk + c];
        sd[j * W + c] = d_out[row * ld_do + head * dk + c];
    }
    __syncthreads();
    for (int j = warp; j < rpi; j += nw) {
        const long item = row_of(j) * heads + head;
        const long item_local = ((long)img * rpi1 + (j % rpi1)) * heads + head;
        const uint32_t tstep = step + (uint32_t)(j / rpi1);
        float dot = 0.f;
        for (int r = lane; r < R; r += 32) {
            const float pr = probs[item * R + r];
            const float D = drop_scale(seed, site, tstep, (uint32_t)(item_local * R + r), p_drop);
            float s = 0.f;
            for (int c = 0; c < dk; ++c) s = fmaf(sd[j * W + c], sv[r * W + c], s);
            const float dp = s * D;
            PD[j * R + r] = pr * D;
            DS[j * R + r] = dp;
            dot = fmaf(pr, dp, dot);
        }
        dot = wsum(dot);
        __syncwarp();
        for (int r = lane; r < R; r += 32) DS[j * R + r] = probs[item * R + r] * (DS[j * R + r] - dot) * scale;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < R * dk; i += blockDim.x) {
        const int r = i / dk, c = i % dk;
        const long g = ((long)img * R + r) * ld_dkv + head * dk + c;
        const float ov = dvv[g], ok = dkk[g];            // the read-modify-write's loads are issued before the reduction over the rows
        float av = 0.f, ak = 0.f;
        for (int j = 0; j < rpi; ++j) {
            av = fmaf(PD[j * R + r], sd[j * W + c], av);
            ak = fmaf(DS[j * R + r], sq[j * W + c], ak);
        }
        dvv[g] = ov + av;
        dkk[g] = ok + ak;
    }
    for (int i = threadIdx.x; i < rpi * dk; i += blockDim.x) {
        const int j = i / dk, c = i % dk;
        float a = 0.f;
        for (int r = 0; r < R; ++r) a = fmaf(DS[j * R + r], sk[r * W + c], a);
        dq[row_of(j) * ld_dq + head * dk + c] = a;
    }
}

// d x[img, r, :] += d mean[img, :] / R        (masked: mean over the valid regions, AoAModel.py:216-219 -> += mask[r] * d mean / sum(mask))
__global__ void mean_backward_kernel(int R, int H, const float* __restrict__ d_mean, long ld_dm, float* __restrict__ dx, long ld_dx,
                                     const float* __restrict__ mask, long ld_mask) {
    const int row = blockIdx.x;              // img * R + r
    const int img = row / R, r = row % R;
    float inv = 1.0f / (float)R;
    if (mask != nullptr) {
        float cnt = 0.f;
        for (int j = 0; j < R; ++j) cnt += mask[(long)img * ld_mask + j];
        inv = mask[(long)img * ld_mask + r] / cnt;
    }
    for (int c = threadIdx.x; c < H; c += blockDim.x) dx[(long)row * ld_dx + c] += d_mean[(long)img * ld_dm + c] * inv;
}

// out[r, :] = a[r, :] + b[r, :] * dropmask(site, step, r*cols + c)      (SublayerConnection: x + dropout(sublayer(norm(x))))
__global__ void add_dropout_kernel(int rows, int cols, const float* __restrict__ a, long ld_a, const float* __restrict__ b, long ld_b, float* __restrict__ out,
                                   long ld_o, unsigned long long seed, uint32_t site, uint32_t step, float p) {
    const long n = (long)rows * cols;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const long r = i / cols;
        const int c = (int)(i % cols);
        out[r * ld_o + c] = a[r * ld_a + c] + b[r * ld_b + c] * drop_scale(seed, site, step, (uint32_t)i, p);
    }
}

// out[r, c] = (c < c1 ? a[r, c] : b[r, c - c1]) * dropmask(site, step, r*(c1+c2) + c)     (dropout_aoa(cat[x, query]))
__global__ void cat_dropout_kernel(int rows, int c1, int c2, const float* __restrict__ a, long ld_a, const float* __restrict__ b, long ld_b,
                                   float* __restrict__ out, long ld_o, unsigned long long seed, uint32_t site, uint32_t step, float p) {
    const int cols = c1 + c2;
    const long n = (long)rows * cols;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const long r = i / cols;
        const int c = (int)(i % cols);
        const float v = c < c1 ? a[r * ld_a + c] : b[r * ld_b + (c - c1)];
        out[r * ld_o + c] = v * drop_scale(seed, site, step, (uint32_t)i, p);
    }
}

int blocks_for(long n) {
    long b = (n + 255) / 256;
    return (int)(b < 1 ? 1 : (b > sm_count() * 16 ? sm_count() * 16 : b));
}

}  // namespace

#define LAUNCH_OK() do { CAPB_CHECK_CUDA(cudaGetLastError()); return 0; } while (0)

int ln_backward_launch(int rows, int D, const float* x, long ld_x, const float* a, const float* dy, long ld_dy, float eps, float* dx, long ld_dx, int accumulate,
                       float* stats, float* da, float* db, int accumulate_params, cudaStream_t st, const float* add1, long ld_a1, const float* add2, long ld_a2) {
    ln_backward_kernel<<<rows, 128, 0, st>>>(rows, D, x, ld_x, a, dy, ld_dy, eps, dx, ld_dx, accumulate, reinterpret_cast<float2*>(stats), add1, ld_a1, add2, ld_a2);
    CAPB_CHECK_CUDA(cudaGetLastError());
    ln_param_grad_kernel<<<cdiv(D, 32), 256, 0, st>>>(rows, D, x, ld_x, dy, ld_dy, reinterpret_cast<const float2*>(stats), da, db, accumulate_params);
    LAUNCH_OK();
}
int glu_backward_launch(int rows, int H, const float* t, long ld_t, const float* dy, long ld_dy, float* dt, long ld_dt, cudaStream_t st) {
    glu_backward_kernel<<<blocks_for((long)rows * H), 256, 0, st>>>(rows, H, t, ld_t, dy, ld_dy, dt, ld_dt);
    LAUNCH_OK();
}
inline int attn_chunks(int seqs, int heads, int units) {      // query chunks so that the grid reaches about two CTAs per SM
    int z = (296 + seqs * heads - 1) / (seqs * heads);
    if (z > 4) z = 4;
    if (z > units) z = units;
    return z < 1 ? 1 : z;
}
int seq_attn_train_launch(int seqs, int n_keys, int q_lo, int q_hi, int heads, int dk, int causal, int idx_L, long b_stride, long p_stride, const float* q,
                          const float* k, const float* v, long ld, unsigned long long seed, int site, float p, float* out, long ld_out, const float* key_mask,
                          long ld_mask, cudaStream_t st, int form) {
    if (seqs <= 0 || q_hi <= q_lo) return 0;
    CAPB_REQUIRE((dk & 3) == 0, "self-attention (train): the head width must be a multiple of 4");
    const size_t smem = sizeof(float) * ((size_t)2 * n_keys * (dk + 4) + 8 * n_keys + 8 * dk);
    if (form == 2 || (form == 0 && smem > 200 * 1024)) {
        ActView o;
        o.f = out; o.ld = ld_out;
        return attn_tiled_forward_launch(seqs, n_keys, heads, dk, idx_L, b_stride, p_stride, q, k, v, ld, key_mask, ld_mask, seed, site, p, o, st, causal,
                                         q_lo, q_hi);
    }
    CAPB_REQUIRE(smem <= 200 * 1024, "self-attention (train): keys * head width too large for the shared-memory staging");
    static std::atomic<unsigned long long> configured{0};
    if (first_use_on_device(configured)) {
        CAPB_CHECK_CUDA(cudaFuncSetAttribute(seq_attn_train_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    }
    SeqAttn a;
    a.n_keys = n_keys; a.dk = dk; a.heads = heads; a.q_lo = q_lo; a.q_hi = q_hi; a.causal = causal; a.idx_L = idx_L; a.b_stride = b_stride; a.p_stride = p_stride;
    a.ld = ld; a.scale = 1.0f / sqrtf((float)dk); a.p_drop = p; a.seed = seed; a.site = (uint32_t)site; a.key_mask = key_mask; a.ld_mask = ld_mask;
    seq_attn_train_kernel<<<dim3(seqs, heads, attn_chunks(seqs, heads, q_hi - q_lo)), 256, smem, st>>>(a, q, k, v, out, ld_out);
    LAUNCH_OK();
}
int seq_attn_backward_launch(int seqs, int n_keys, int heads, int dk, int causal, int idx_L, long b_stride, long p_stride, const float* q, const float* k,
                             const float* v, long ld, unsigned long long seed, int site, float p, const float* d_out, long ld_do, float* dq, float* dk_,
                             float* dv, long ld_d, const float* key_mask, long ld_mask, cudaStream_t st, int form) {
    if (seqs <= 0) return 0;
    CAPB_REQUIRE((dk & 3) == 0, "self-attention backward: the head width must be a multiple of 4");
    const size_t smem = sizeof(float) * ((size_t)4 * n_keys * (dk + 4) + 2 * n_keys * n_keys);
    if (form == 2 || (form == 0 && smem > 200 * 1024)) {
        return attn_tiled_self_backward_launch(seqs, n_keys, heads, dk, idx_L, b_stride, p_stride, q, k, v, ld, seed, site, p, d_out, ld_do, dq, dk_, dv, ld_d,
                                               key_mask, ld_mask, st, causal);
    }
    CAPB_REQUIRE(smem <= 200 * 1024, "self-attention backward: shared-memory footprint too large");
    static std::atomic<unsigned long long> configured{0};
    if (first_use_on_device(configured)) {
        CAPB_CHECK_CUDA(cudaFuncSetAttribute(seq_attn_backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    }
    SeqAttn a;
    a.n_keys = n_keys; a.dk = dk; a.heads = heads; a.q_lo = 0; a.q_hi = n_keys; a.causal = causal; a.idx_L = idx_L; a.b_stride = b_stride; a.p_stride = p_stride;
    a.ld = ld; a.scale = 1.0f / sqrtf((float)dk); a.p_drop = p; a.seed = seed; a.site = (uint32_t)site; a.key_mask = key_mask; a.ld_mask = ld_mask;
    // every chunk CTA rebuilds P and dS (half of the kernel's work) and owns a whole SM (up to 150 KB of shared memory): chunks only help while
    // the grid stays within one wave (measured: 4 chunks at 80 (image, head) pairs = 320 CTAs took 108 us, 1 chunk 72 us)
    int z = sm_count() / (seqs * heads);
    z = z < 1 ? 1 : (z > 4 ? 4 : z);
    seq_attn_backward_kernel<<<dim3(seqs, heads, z), 256, smem, st>>>(a, q, k, v, d_out, ld_do, dq, dk_, dv, ld_d);
    LAUNCH_OK();
}
// the refiner / encoder form: sequences = images, keys = queries = the R regions, rows image-major
int enc_attn_train_launch(int B, int R, int heads, int dk, const float* q, const float* k, const float* v, long ld, unsigned long long seed, int site, float p,
                          float* out, long ld_out, cudaStream_t st, const float* mask, long ld_mask) {
    return seq_attn_train_launch(B, R, 0, R, heads, dk, 0, R, R, 1, q, k, v, ld, seed, site, p, out, ld_out, mask, ld_mask, st);
}
int enc_attn_backward_launch(int B, int R, int heads, int dk, const float* q, const float* k, const float* v, long ld, unsigned long long seed, int site, float p,
                             const float* d_out, long ld_do, float* dq, float* dk_, float* dv, long ld_d, cudaStream_t st, const float* mask, long ld_mask) {
    return seq_attn_backward_launch(B, R, heads, dk, 0, R, R, 1, q, k, v, ld, seed, site, p, d_out, ld_do, dq, dk_, dv, ld_d, mask, ld_mask, st);
}
int cross_attn_train_launch(int rows, int rpi, int heads, int dk, int R, const float* q, long ld_q, const float* kk, const float* vv, long ld_kv,
                            unsigned long long seed, int site, int step, float p, float* out, long ld_out, float* probs, cudaStream_t st, const float* mask,
                            long ld_mask, int row_mod) {
    CAPB_REQUIRE(dk <= 256, "attention: head width above 256");
    if (rows <= 0) return 0;
    cross_attn_train_kernel<<<rows * heads, 128, sizeof(float) * R, st>>>(rows, rpi, heads, dk, R, q, ld_q, kk, vv, ld_kv, 1.0f / sqrtf((float)dk),
                                                                                        seed, (uint32_t)site, (uint32_t)step, p, out, ld_out, probs, mask, ld_mask,
                                                                                        row_mod > 0 ? row_mod : rows);
    LAUNCH_OK();
}
int cross_attn_backward_launch(int B, int rpi, int heads, int dk, int R, const float* q, long ld_q, const float* kk, const float* vv, long ld_kv,
                               unsigned long long seed, int site, int step, float p, const float* probs, const float* d_out, long ld_do, float* dq, long ld_dq,
                               float* dkk, float* dvv, long ld_dkv, cudaStream_t st, int n_steps, int row_mod, int form) {
    const int rpi1 = rpi;
    rpi = rpi1 * (n_steps > 0 ? n_steps : 1);          // all of the image's rows in this launch
    const size_t smem = sizeof(float) * ((size_t)2 * R * (dk + 1) + 2 * rpi * (dk + 1) + 2 * (size_t)rpi * R);
    if (form == 2 || (form == 0 && smem > 200 * 1024))
        return attn_tiled_cross_backward_launch(B, rpi1, rpi / rpi1, row_mod > 0 ? row_mod : B * rpi1, heads, dk, R, q, ld_q, kk, vv, ld_kv, seed, site, step, p,
                                                probs, d_out, ld_do, dq, ld_dq, dkk, dvv, ld_dkv, st);
    CAPB_REQUIRE(smem <= 200 * 1024, "decoder attention backward: shared-memory footprint too large");
    static std::atomic<unsigned long long> configured{0};
    if (first_use_on_device(configured)) {
        CAPB_CHECK_CUDA(cudaFuncSetAttribute(cross_attn_backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    }
    // 512 threads: the kernel is a chain of global-load rounds (K, V, q, d_out, the dK / dV read-modify-write) on only B x heads CTAs
    cross_attn_backward_kernel<<<dim3(B, heads), 512, smem, st>>>(rpi, heads, dk, R, q, ld_q, kk, vv, ld_kv, 1.0f / sqrtf((float)dk), seed, (uint32_t)site,
                                                                   (uint32_t)step, p, probs, d_out, ld_do, dq, ld_dq, dkk, dvv, ld_dkv, rpi1, row_mod > 0 ? row_mod : B * rpi1);
    LAUNCH_OK();
}
int mean_backward_launch(int B, int R, int H, const float* d_mean, long ld_dm, float* dx, long ld_dx, cudaStream_t st, const float* mask, long ld_mask) {
    mean_backward_kernel<<<B * R, 256, 0, st>>>(R, H, d_mean, ld_dm, dx, ld_dx, mask, ld_mask);
    LAUNCH_OK();
}
int add_dropout_launch(int rows, int cols, const float* a, long ld_a, const float* b, long ld_b, float* out, long ld_o, unsigned long long seed, int site, int step,
                       float p, cudaStream_t st) {
    add_dropout_kernel<<<blocks_for((long)rows * cols), 256, 0, st>>>(rows, cols, a, ld_a, b, ld_b, out, ld_o, seed, (uint32_t)site, (uint32_t)step, p);
    LAUNCH_OK();
}
int cat_dropout_launch(int rows, int c1, int c2, const float* a, long ld_a, const float* b, long ld_b, float* out, long ld_o, unsigned long long seed, int site,
                       int step, float p, cudaStream_t st) {
    cat_dropout_kernel<<<blocks_for((long)rows * (c1 + c2)), 256, 0, st>>>(rows, c1, c2, a, ld_a, b, ld_b, out, ld_o, seed, (uint32_t)site, (uint32_t)step, p);
    LAUNCH_OK();
}
int aoa_step_inputs_launch(int rows, int E, int H, int rpi, const int* tok_src, int* tok_dst, const float* emb, float* xt, const float* mean, long ld_mean,
                           const float* out_prev, float* x1c, unsigned long long seed, int step, float p_lm, float p_ctx, cudaStream_t st) {
    if (rows <= 0) return 0;
    aoa_step_inputs_kernel<<<rows, 256, 0, st>>>(E, H, rpi, tok_src, tok_dst, emb, xt, mean, ld_mean, out_prev, x1c, seed, (uint32_t)step, p_lm, p_ctx);
    LAUNCH_OK();
}
int glu_dropout_launch(int rows, int H, const float* t, long ld_t, float* out, long ld_o, float* outd, long ld_d, unsigned long long seed, int step, float p,
                       cudaStream_t st) {
    if (rows <= 0) return 0;
    glu_dropout_kernel<<<blocks_for((long)rows * H), 256, 0, st>>>(rows, H, t, ld_t, out, ld_o, outd, ld_d, seed, (uint32_t)step, p);
    LAUNCH_OK();
}
int glu_backward_fused_launch(int rows, int H, const float* t, long ld_t, const float* d_outd, long ld_dd, const float* dctx, float* dt, long ld_dt,
                              unsigned long long seed, int step, float p, cudaStream_t st) {
    if (rows <= 0) return 0;
    glu_backward_fused_kernel<<<blocks_for((long)rows * H), 256, 0, st>>>(rows, H, t, ld_t, d_outd, ld_dd, dctx, dt, ld_dt, seed, (uint32_t)step, p);
    LAUNCH_OK();
}

CAPB_DEFINE_SALT_SETTER(dropout_salt_set_aoa)

}  // namespace capb200
