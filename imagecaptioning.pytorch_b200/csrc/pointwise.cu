// Element-wise / small-reduction kernels of the per-timestep core.
//
//   state_gather_embed   embedding lookup (+ReLU) and parent-beam state reorder   AttModel.py:168 (embed), CaptionModel.py:105-108
//   lstm_pointwise       nn.LSTMCell gate math (i,f,g,o)                          AttModel.py:628,635
//   maxout_pointwise     NewFC maxout LSTM core                                   FCModel.py:25-42
//   additive_attention   softmax_r(w . tanh(p_att[r] + W_h h)) then sum_r a_r v_r AttModel.py:728-748
//
// All kernels read per-IMAGE features (p_att, att) by row / rows_per_image instead of the beam-replicated copies the
// reference materialises with repeat_tensors (AttModel.py:241-243).
#include "common.cuh"
#include "kernels.cuh"

namespace capb200 {

static int pw_blocks(long total) {
    long b = (total + 255) / 256;
    return (int)(b > sm_count() * 8 ? sm_count() * 8 : b);
}

namespace {

__device__ __forceinline__ float sigmoidf_(float x) { return fast_sigmoid(x); }

__device__ __forceinline__ void store_act(const ActView& o, long row, int col, float v) {
    o.f[row * o.ld + col] = v;
    if (o.hi != nullptr) {
        __half h, l;
        split_f32(v, h, l);
        o.hi[row * o.ld + col] = h;
        o.lo[row * o.ld + col] = l;
    }
}

// grid = rows, block = 256.  src_row < 0 means "fresh zero state" (first step).
__global__ void state_gather_embed_kernel(int rows, const int* __restrict__ tokens, const int* __restrict__ src_row,
                                          const float* __restrict__ emb, long ld_emb, int E, int relu, ActView xt,
                                          int H, int nstate, StateCopy sc0, StateCopy sc1) {
    const int r = blockIdx.x;
    if (r >= rows) return;
    const int tok = tokens[r];
    const float* e = emb + (long)tok * ld_emb;
    for (int c = threadIdx.x; c < E; c += blockDim.x) {
        float v = __ldg(e + c);
        if (relu) v = fmaxf(v, 0.f);
        store_act(xt, r, c, v);
    }
    const int src = src_row ? src_row[r] : r;
    const bool vec = (H & 3) == 0 && (sc0.ld_src & 3) == 0 && (sc0.dst.ld & 3) == 0 && (nstate < 2 || ((sc1.ld_src & 3) == 0 && (sc1.dst.ld & 3) == 0));
    if (vec) {
        // 128-bit copies with the loads of both states issued before any store (the scalar loop was latency-bound: r01f capture)
        for (int c4 = threadIdx.x; c4 < (H >> 2); c4 += blockDim.x) copy_states4(r, src, c4, nstate, sc0, sc1);
        return;
    }
    for (int s = 0; s < nstate; ++s) {
        const StateCopy& sc = (s == 0) ? sc0 : sc1;
        for (int c = threadIdx.x; c < H; c += blockDim.x) {
            const float v = (src < 0) ? 0.f : sc.src[(long)src * sc.ld_src + c];
            store_act(sc.dst, r, c, v);
        }
    }
}

// gates [rows, 4H] in the nn.LSTMCell order i,f,g,o (bias already added by the GEMM epilogue).
// gather_bias (optional): per-token gate contribution table[token[r], 4H] added before the non-linearities.
__global__ void lstm_pointwise_kernel(int rows, int H, const float* __restrict__ gates, long ld_g, const int* __restrict__ src_row,
                                      const float* __restrict__ c_prev, long ld_cp, float* __restrict__ c_out, long ld_co, ActView h_out,
                                      const float* __restrict__ gather_bias, long ld_gb, const int* __restrict__ gather_idx) {
    const long total = (long)rows * H;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int r = (int)(i / H), c = (int)(i % H);
        const float* g = gates + (long)r * ld_g;
        float gi = g[c], gf = g[H + c], gg = g[2 * H + c], go = g[3 * H + c];
        if (gather_bias != nullptr) {
            const float* gb = gather_bias + (long)gather_idx[r] * ld_gb;
            gi += __ldg(gb + c); gf += __ldg(gb + H + c); gg += __ldg(gb + 2 * H + c); go += __ldg(gb + 3 * H + c);
        }
        const int src = src_row ? src_row[r] : r;
        const float cp = (src < 0 || c_prev == nullptr) ? 0.f : c_prev[(long)src * ld_cp + c];
        const float cn = sigmoidf_(gf) * cp + sigmoidf_(gi) * fast_tanh(gg);
        const float hn = sigmoidf_(go) * fast_tanh(cn);
        c_out[(long)r * ld_co + c] = cn;
        store_act(h_out, r, c, hn);
    }
}

// LSTM cell + the LayerNorm of its output in one launch (AoANet decoder: core.attention.norm(h_att) follows the cell, AoAModel.py:166-168),
// one CTA of 256 threads per row, H <= 2048: the cell of lstm_pointwise_kernel (same expressions), h kept in registers for the two
// reductions of TransformerModel.LayerNorm (unbiased std, eps added to std).
__global__ void __launch_bounds__(256) lstm_ln_kernel(int H, const float* __restrict__ gates, long ld_g, const float* __restrict__ c_prev, long ld_cp,
                                                      float* __restrict__ c_out, long ld_co, float* __restrict__ h_out, long ld_h, const float* __restrict__ ln_a,
                                                      const float* __restrict__ ln_b, float eps, float* __restrict__ ln_out, long ld_ln) {
    __shared__ float sh[8];
    const int r = blockIdx.x;
    const float* g = gates + (long)r * ld_g;
    float hv[8];
    float s = 0.f;
#pragma unroll
    for (int u = 0; u < 8; ++u) {
        const int c = threadIdx.x + 256 * u;
        hv[u] = 0.f;
        if (c < H) {
            const float gi = g[c], gf = g[H + c], gg = g[2 * H + c], go = g[3 * H + c];
            const float cp = c_prev == nullptr ? 0.f : c_prev[(long)r * ld_cp + c];
            const float cn = sigmoidf_(gf) * cp + sigmoidf_(gi) * fast_tanh(gg);
            const float hn = sigmoidf_(go) * fast_tanh(cn);
            c_out[(long)r * ld_co + c] = cn;
            h_out[(long)r * ld_h + c] = hn;
            hv[u] = hn;
            s += hn;
        }
    }
    auto bsum = [&](float v) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        __syncthreads();
        if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
        __syncthreads();
        return ((sh[0] + sh[1]) + (sh[2] + sh[3])) + ((sh[4] + sh[5]) + (sh[6] + sh[7]));
    };
    const float mean = bsum(s) / (float)H;
    float q = 0.f;
#pragma unroll
    for (int u = 0; u < 8; ++u) { const int c = threadIdx.x + 256 * u; if (c < H) { const float d = hv[u] - mean; q = fmaf(d, d, q); } }
    const float stdv = sqrtf(bsum(q) / (float)(H - 1));
    const float inv = 1.0f / (stdv + eps);
#pragma unroll
    for (int u = 0; u < 8; ++u) { const int c = threadIdx.x + 256 * u; if (c < H) ln_out[(long)r * ld_ln + c] = __ldg(ln_a + c) * (hv[u] - mean) * inv + __ldg(ln_b + c); }
}

// sums [rows, 5H]: sigmoid(i), sigmoid(f), sigmoid(o), then two candidates whose max is the cell input.
__global__ void maxout_pointwise_kernel(int rows, int H, const float* __restrict__ sums, long ld_s, const int* __restrict__ src_row,
                                        const float* __restrict__ c_prev, long ld_cp, float* __restrict__ c_out, long ld_co, ActView h_out) {
    const long total = (long)rows * H;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int r = (int)(i / H), c = (int)(i % H);
        const float* s = sums + (long)r * ld_s;
        const float gi = sigmoidf_(s[c]), gf = sigmoidf_(s[H + c]), go = sigmoidf_(s[2 * H + c]);
        const float gg = fmaxf(s[3 * H + c], s[4 * H + c]);
        const int src = src_row ? src_row[r] : r;
        const float cp = (src < 0 || c_prev == nullptr) ? 0.f : c_prev[(long)src * ld_cp + c];
        const float cn = gf * cp + gi * gg;
        const float hn = go * fast_tanh(cn);
        c_out[(long)r * ld_co + c] = cn;
        store_act(h_out, r, c, hn);
    }
}

// Additive attention in two launches sized for the whole chip:
//   att_score_kernel    one WARP per (image, region): score[row, r] = w . tanh(p_att[img, r, :] + att_h[row, :]) + b for the image's
//                       rows (beams / samples); p_att is read once per warp, never replicated per beam.
//   att_combine_kernel  one CTA per (image, 256-column slice): softmax over regions (+ mask renormalisation), then
//                       out[row, c] = sum_r a[row, r] * att[img, r, c].
// tanh is evaluated as 1 - 2 / (1 + exp(2x)) on the SFU (ex2.approx): absolute error < 3e-7, far below the 1e-4 log-prob bar.
constexpr int ATT_JB = 5;       // rows handled per pass (beam 5 = one pass)
constexpr int ATT_SW = 8;       // warps (= regions) per CTA
// grid = (ceil(R / 8), B): the CTA stages the image's att_h rows in shared memory once (coalesced), then each warp scores one region.
// NA = ceil(A / 32) rounded up to a power of two is a template parameter so the inner loops are branch-free and the
// independent tanh chains of different k overlap (the runtime-bound version serialised them).
template <int NA>
__global__ void __launch_bounds__(ATT_SW * 32, NA <= 16 ? 5 : 2) att_score_kernel(int rpi, int R, int A, const float* __restrict__ att_h, long ld_ah,
                                                                const float* __restrict__ p_att, long ld_pa, const float* __restrict__ alpha_w,
                                                                const float* __restrict__ alpha_b_ptr, float* __restrict__ score) {
    // tanh(x) = 1 - 2 / (1 + 2^(x * 2 log2 e)): p_att and att_h are pre-multiplied by 2 log2(e) when loaded, the sum over a of
    // w[a] * tanh = sum(w) - 2 * sum_a w[a] / (1 + 2^z), and four reciprocals share one MUFU.RCP (1/y_i from 1/(y0 y1 y2 y3)).
    // The r01f capture showed the earlier version issue-bound at 23 instructions per tanh; this form needs about 10.
    // Registers: five CTAs per SM (<= 51 registers) turn the 1280-CTA grid of the headline shape from 3 rounds into 2, so the
    // attention weights w live in shared memory instead of 16 registers per lane.
    extern __shared__ float s_ah[];               // [ATT_JB][NA * 32] pre-scaled (zero padded beyond A), then w [NA * 32]
    constexpr int AP = NA * 32;
    float* s_w = s_ah + ATT_JB * AP;
    constexpr float kC = 2.885390081777927f;      // 2 * log2(e)
    const int img = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int r = blockIdx.x * ATT_SW + warp;
    const float alpha_b = __ldg(alpha_b_ptr);
    float pv[NA];                                  // element k = 4 * g + u  <->  hidden index a = 128 * g + 4 * lane + u
    const bool live = r < R;
    const float* pr = p_att + ((long)img * R + (live ? r : 0)) * ld_pa;
    for (int i = threadIdx.x; i < AP; i += ATT_SW * 32) s_w[i] = (i < A) ? __ldg(alpha_w + i) : 0.f;      // zero weight kills padded lanes
    __syncthreads();
    float wsum = 0.f;
#pragma unroll
    for (int k = 0; k < NA; ++k) {
        const int a = (NA % 4 == 0) ? 128 * (k >> 2) + 4 * lane + (k & 3) : lane + 32 * k;
        pv[k] = (live && a < A) ? __ldg(pr + a) * kC : 0.f;
        wsum += s_w[a];
    }
    for (int j0 = 0; j0 < rpi; j0 += ATT_JB) {
        const int nj = min(ATT_JB, rpi - j0);
        __syncthreads();
        for (int i = threadIdx.x; i < nj * AP; i += ATT_SW * 32) {
            const int j = i / AP, a = i - j * AP;
            s_ah[i] = (a < A) ? att_h[((long)img * rpi + j0 + j) * ld_ah + a] * kC : 0.f;
        }
        __syncthreads();
        if (live) {
            float part[ATT_JB];
#pragma unroll
            for (int j = 0; j < ATT_JB; ++j) {
                part[j] = 0.f;
                if (j < nj) {
                    if (NA % 4 == 0) {
                        float acc = 0.f;
#pragma unroll
                        for (int g = 0; g < NA / 4; ++g) {
                            const float4 ah = *reinterpret_cast<const float4*>(&s_ah[j * AP + 128 * g + 4 * lane]);
                            const float z[4] = {pv[4 * g] + ah.x, pv[4 * g + 1] + ah.y, pv[4 * g + 2] + ah.z, pv[4 * g + 3] + ah.w};
                            float y[4];
#pragma unroll
                            for (int u = 0; u < 4; ++u) {
                                float e;
                                asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(fminf(z[u], 28.0f)));      // 2^28: tanh rounds to 1 long before
                                y[u] = 1.0f + e;
                            }
                            const float p01 = y[0] * y[1], p23 = y[2] * y[3];
                            float rr;
                            asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(rr) : "f"(p01 * p23));
                            const float r01 = rr * p23, r23 = rr * p01;
                            const float4 w4 = *reinterpret_cast<const float4*>(&s_w[128 * g + 4 * lane]);
                            acc = fmaf(w4.x, r01 * y[1], acc);
                            acc = fmaf(w4.y, r01 * y[0], acc);
                            acc = fmaf(w4.z, r23 * y[3], acc);
                            acc = fmaf(w4.w, r23 * y[2], acc);
                        }
                        part[j] = fmaf(-2.0f, acc, wsum);
                    } else {
#pragma unroll
                        for (int k = 0; k < NA; ++k) {
                            float e;
                            asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(fminf(pv[k] + s_ah[j * AP + lane + 32 * k], 28.0f)));
                            part[j] = fmaf(s_w[lane + 32 * k], 1.0f - __fdividef(2.0f, 1.0f + e), part[j]);
                        }
                    }
                }
            }
#pragma unroll
            for (int j = 0; j < ATT_JB; ++j) {
                float v = part[j];
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
                if (lane == 0 && j < nj) score[((long)img * rpi + j0 + j) * R + r] = v + alpha_b;
            }
        }
    }
}

// (A one-launch fusion of the two kernels -- one CTA of 16 warps per image: scores, softmax, weighted sum -- was measured in round 2: no faster
// than the pair at 256 images x 5 beams (6.08 vs 6.08 ms per batch; 36 regions on 16 warps leave the score phase at 75 % utilisation and the
// image count, not the chip, sets the parallelism), so the split form stays.)
constexpr int ATT_CT = 256;
__global__ void __launch_bounds__(ATT_CT) att_combine_kernel(int rpi, int R, int H, const float* __restrict__ score, const float* __restrict__ att,
                                                             long ld_at, const float* __restrict__ mask, long ld_mask, ActView out,
                                                             float* __restrict__ alpha_out) {
    extern __shared__ float s_w[];                 // [ATT_JB][R]
    const int img = blockIdx.x;
    const int c = blockIdx.y * ATT_CT + threadIdx.x;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int j0 = 0; j0 < rpi; j0 += ATT_JB) {
        const int nj = min(ATT_JB, rpi - j0);
        __syncthreads();
        if (warp < nj) {                            // softmax over the regions of one row per warp
            const float* sc = score + ((long)img * rpi + j0 + warp) * R;
            float* w = s_w + warp * R;
            float mx = -INFINITY;
            for (int r = lane; r < R; r += 32) mx = fmaxf(mx, sc[r]);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
            float sum = 0.f;
            for (int r = lane; r < R; r += 32) { const float e = expf(sc[r] - mx); w[r] = e; sum += e; }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
            const float inv = 1.0f / sum;
            float msum = 0.f;
            for (int r = lane; r < R; r += 32) {
                float v = w[r] * inv;
                if (mask != nullptr) { v *= mask[(long)img * ld_mask + r]; msum += v; }
                w[r] = v;
            }
            if (mask != nullptr) {
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) msum += __shfl_xor_sync(0xffffffffu, msum, o);
                for (int r = lane; r < R; r += 32) w[r] = w[r] / msum;
            }
        }
        __syncthreads();
        if (alpha_out != nullptr && blockIdx.y == 0) {       // training keeps the attention weights for the backward pass
            for (int i = threadIdx.x; i < nj * R; i += ATT_CT) alpha_out[((long)img * rpi + j0) * R + i] = s_w[i];
        }
        if (c < H) {
            float acc[ATT_JB];
#pragma unroll
            for (int j = 0; j < ATT_JB; ++j) acc[j] = 0.f;
            const float* ap = att + (long)img * R * ld_at + c;
            // (batching several feature loads per thread was measured twice and is slower: 14.5 -> 17-20 us)
            for (int r = 0; r < R; ++r) {
                const float v = __ldg(ap + (long)r * ld_at);
#pragma unroll
                for (int j = 0; j < ATT_JB; ++j)
                    if (j < nj) acc[j] = fmaf(s_w[j * R + r], v, acc[j]);
            }
#pragma unroll
            for (int j = 0; j < ATT_JB; ++j)
                if (j < nj) store_act(out, (long)img * rpi + j0 + j, c, acc[j]);
        }
    }
}

__global__ void relu_copy_kernel(const float* __restrict__ x, long n, ActView out_flat) {
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const float v = fmaxf(__ldg(x + i), 0.f);
        out_flat.f[i] = v;
        if (out_flat.hi) { __half h, l; split_f32(v, h, l); out_flat.hi[i] = h; out_flat.lo[i] = l; }
    }
}

}  // namespace

int relu_copy_launch(const float* x, long n, ActView out_flat, cudaStream_t stream) {
    relu_copy_kernel<<<pw_blocks(n), 256, 0, stream>>>(x, n, out_flat);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int state_gather_embed_launch(int rows, const int* tokens, const int* src_row, const float* emb, long ld_emb, int E, int relu,
                              ActView xt, int H, int nstate, StateCopy sc0, StateCopy sc1, cudaStream_t stream) {
    if (rows <= 0) return 0;
    state_gather_embed_kernel<<<rows, 256, 0, stream>>>(rows, tokens, src_row, emb, ld_emb, E, relu, xt, H, nstate, sc0, sc1);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}


int lstm_pointwise_launch(int rows, int H, const float* gates, long ld_g, const int* src_row, const float* c_prev, long ld_cp,
                          float* c_out, long ld_co, ActView h_out, const float* gather_bias, long ld_gb, const int* gather_idx,
                          cudaStream_t stream) {
    if (rows <= 0) return 0;
    lstm_pointwise_kernel<<<pw_blocks((long)rows * H), 256, 0, stream>>>(rows, H, gates, ld_g, src_row, c_prev, ld_cp, c_out, ld_co, h_out,
                                                                          gather_bias, ld_gb, gather_idx);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int lstm_ln_launch(int rows, int H, const float* gates, long ld_g, const float* c_prev, long ld_cp, float* c_out, long ld_co, float* h_out, long ld_h,
                   const float* ln_a, const float* ln_b, float eps, float* ln_out, long ld_ln, cudaStream_t stream) {
    if (rows <= 0) return 0;
    CAPB_REQUIRE(H <= 2048, "lstm_ln: hidden size above 2048");
    lstm_ln_kernel<<<rows, 256, 0, stream>>>(H, gates, ld_g, c_prev, ld_cp, c_out, ld_co, h_out, ld_h, ln_a, ln_b, eps, ln_out, ld_ln);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int maxout_pointwise_launch(int rows, int H, const float* sums, long ld_s, const int* src_row, const float* c_prev, long ld_cp,
                            float* c_out, long ld_co, ActView h_out, cudaStream_t stream) {
    if (rows <= 0) return 0;
    maxout_pointwise_kernel<<<pw_blocks((long)rows * H), 256, 0, stream>>>(rows, H, sums, ld_s, src_row, c_prev, ld_cp, c_out, ld_co, h_out);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int additive_attention_launch(int n_images, int rpi, int R, int A, int H, const float* att_h, long ld_ah, const float* p_att, long ld_pa,
                              const float* att, long ld_at, const float* mask, long ld_mask, const float* alpha_w, const float* alpha_b,
                              float* score_scratch, ActView out, cudaStream_t stream, float* alpha_out) {
    if (n_images <= 0 || rpi <= 0) return 0;
    CAPB_REQUIRE(A <= 1024, "attention: att_hid_size above 1024");
    CAPB_REQUIRE(score_scratch != nullptr, "attention: score scratch missing");
    const int na = cdiv(A, 32);
    dim3 sgrid(cdiv(R, ATT_SW), n_images);
#define CAPB_ATT_CASE(NA_)                                                                                                             \
    att_score_kernel<NA_><<<sgrid, ATT_SW * 32, sizeof(float) * (ATT_JB + 1) * NA_ * 32, stream>>>(rpi, R, A, att_h, ld_ah, p_att, ld_pa, alpha_w, \
                                                                                               alpha_b, score_scratch)
    if (na <= 2) CAPB_ATT_CASE(2);
    else if (na <= 4) CAPB_ATT_CASE(4);
    else if (na <= 8) CAPB_ATT_CASE(8);
    else if (na <= 16) CAPB_ATT_CASE(16);
    else CAPB_ATT_CASE(32);
#undef CAPB_ATT_CASE
    CAPB_CHECK_CUDA(cudaGetLastError());
    const size_t smem = sizeof(float) * (size_t)ATT_JB * R;
    CAPB_REQUIRE(smem <= 48 * 1024, "attention: too many regions");
    dim3 grid(n_images, cdiv(H, ATT_CT));
    att_combine_kernel<<<grid, ATT_CT, smem, stream>>>(rpi, R, H, score_scratch, att, ld_at, mask, ld_mask, out, alpha_out);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace capb200
