// Kernels for the Transformer captioner (and shared with AoA): custom LayerNorm, token embedding + positional encoding,
// encoder self-attention, KV-cached decoder self-attention (with beam ancestry) and per-image cross-attention.
//
//   layer_norm          captioning/models/TransformerModel.py:76-87    a*(x-mean)/(std_unbiased+eps)+b, eps = 1e-6
//   embed_pe            TransformerModel.py:208-235                     lut[tok]*sqrt(d_model) + pe[t]
//   enc_self_attention  TransformerModel.py:152-195 (encoder use, mask [B,1,R])
//   dec_self_attention  TransformerModel.py:351-363: the reference re-runs all t tokens every step; with a causal mask the
//                       K/V of earlier positions never change, so they are cached per (layer, step, row) and a row reads its
//                       ancestors' entries through the beam history (no cache reordering by parent beam)
//   cross_attention     src_attn over the image's encoder memory; K/V are per IMAGE, rows index them by row / rows_per_image
#include "../../include/capb200.h"
#include "common.cuh"
#include "kernels.cuh"
#include "attn.cuh"

namespace capb200 {

namespace {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

__device__ __forceinline__ void store_act2(const ActView& o, long row, int col, float v) {
    o.f[row * o.ld + col] = v;
    if (o.hi != nullptr) {
        __half h, l;
        split_f32(v, h, l);
        o.hi[row * o.ld + col] = h;
        o.lo[row * o.ld + col] = l;
    }
}

// one warp per row
// One CTA of 128 threads per row (the rows are few -- 10 .. 1280 -- and a single warp walking a 1024-wide row three times was latency bound).
__device__ __forceinline__ float block_sum128(float v, float* sh) {
    v = warp_sum(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    return (sh[0] + sh[1]) + (sh[2] + sh[3]);
}
__global__ void __launch_bounds__(128) layer_norm_kernel(int rows, int D, const float* __restrict__ x, long ld_x, const float* __restrict__ a,
                                                         const float* __restrict__ b, float eps, ActView out) {
    __shared__ float sh[4];
    const int row = blockIdx.x;
    const float* xr = x + (long)row * ld_x;
    float s = 0.f;
    for (int c = threadIdx.x; c < D; c += 128) s += xr[c];
    const float mean = block_sum128(s, sh) / (float)D;
    float q = 0.f;
    for (int c = threadIdx.x; c < D; c += 128) { const float d = xr[c] - mean; q = fmaf(d, d, q); }
    const float stdv = sqrtf(block_sum128(q, sh) / (float)(D - 1));      // torch.std: unbiased
    const float inv = 1.0f / (stdv + eps);
    for (int c = threadIdx.x; c < D; c += 128) store_act2(out, row, c, __ldg(a + c) * (xr[c] - mean) * inv + __ldg(b + c));
}

__global__ void embed_pe_kernel(int rows, int D, const int* __restrict__ tokens, const float* __restrict__ lut, const float* __restrict__ pe_row,
                                float scale, ActView out) {
    const int row = blockIdx.x;
    const float* e = lut + (long)tokens[row] * D;
    for (int c = threadIdx.x; c < D; c += blockDim.x) store_act2(out, row, c, __ldg(e + c) * scale + __ldg(pe_row + c));
}

// Encoder / refiner self-attention: one CTA per (image, head); K and V head slices staged in shared memory.
// q,k,v: [B*R, ld] with the head at columns [head*dk, (head+1)*dk).  mask[B, R] (1 = valid key) or nullptr.
__global__ void __launch_bounds__(256) enc_self_attention_kernel(int R, int dk, const float* __restrict__ q, const float* __restrict__ k,
                                                                 const float* __restrict__ v, long ld, const float* __restrict__ mask, long ld_mask,
                                                                 float scale, ActView out) {
    extern __shared__ float sm[];
    float* sk = sm;                 // [R][dk+1]
    float* sv = sk + R * (dk + 1);  // [R][dk+1]
    float* sp = sv + R * (dk + 1);  // [warps][R]
    const int img = blockIdx.x, head = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
#pragma unroll 4
    for (int i = threadIdx.x; i < R * dk; i += blockDim.x) {       // independent coalesced loads, four in flight per thread
        const int r = i / dk, c = i % dk;
        sk[r * (dk + 1) + c] = k[((long)img * R + r) * ld + head * dk + c];
        sv[r * (dk + 1) + c] = v[((long)img * R + r) * ld + head * dk + c];
    }
    __syncthreads();
    float* p = sp + warp * R;
    float* qs = sp + nw * R + warp * dk;                        // this warp's query row
    const int q_lo = (int)(((long)R * blockIdx.z) / gridDim.z), q_hi = (int)(((long)R * (blockIdx.z + 1)) / gridDim.z);   // query chunk of this CTA
    for (int qi = q_lo + warp; qi < q_hi; qi += nw) {
        const float* qr = q + ((long)img * R + qi) * ld + head * dk;
        for (int c = lane; c < dk; c += 32) qs[c] = qr[c];
        __syncwarp();
        float mx = -INFINITY;
        for (int r = lane; r < R; r += 32) {
            float s = 0.f;
            for (int c = 0; c < dk; ++c) s = fmaf(qs[c], sk[r * (dk + 1) + c], s);
            s *= scale;
            if (mask != nullptr && mask[(long)img * ld_mask + r] == 0.f) s = -INFINITY;
            p[r] = s;
            mx = fmaxf(mx, s);
        }
        mx = warp_max(mx);
        float sum = 0.f;
        for (int r = lane; r < R; r += 32) { const float e = expf(p[r] - mx); p[r] = e; sum += e; }
        sum = warp_sum(sum);
        __syncwarp();
        const float inv = 1.0f / sum;
        for (int c = lane; c < dk; c += 32) {
            float acc = 0.f;
            for (int r = 0; r < R; ++r) acc = fmaf(p[r], sv[r * (dk + 1) + c], acc);
            store_act2(out, (long)img * R + qi, head * dk + c, acc * inv);
        }
        __syncwarp();
    }
}

// Decoder self-attention at step t for `rows` rows: one warp per (row, head).
//   qkv      [rows, 3D] this step's projections (q | k | v)
//   kcache   [T][cap_rows][D] keys of earlier steps (this layer), vcache likewise; the kernel also writes step t's k, v into them
//   anc      [rows, ld_anc] ancestor row of each earlier step (nullptr = identity)
__global__ void __launch_bounds__(128) dec_self_attention_kernel(int rows, int heads, int dk, int t, const float* __restrict__ qkv, long ld_qkv,
                                                                 float* __restrict__ kcache, float* __restrict__ vcache, long step_stride, long ld_c,
                                                                 const int* __restrict__ anc, long ld_anc, const long long* __restrict__ labels,
                                                                 long ld_lab, float scale, ActView out) {
    const int item = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (item >= rows * heads) return;
    const int lane = threadIdx.x & 31;
    const int row = item / heads, head = item % heads;
    const int D = heads * dk;
    const float* qr = qkv + (long)row * ld_qkv + head * dk;
    const float* kr = qr + D;
    const float* vr = qr + 2 * D;
    // publish this step's key / value for later steps
    for (int c = lane; c < dk; c += 32) {
        kcache[(long)t * step_stride + (long)row * ld_c + head * dk + c] = kr[c];
        vcache[(long)t * step_stride + (long)row * ld_c + head * dk + c] = vr[c];
    }
    // scores over positions 0..t (lane s handles position s; dec_self_attention_launch runs this kernel only for t < 32)
    float sc = -INFINITY;
    if (lane <= t) {
        const float* ks;
        if (lane == t) ks = kr;
        else {
            const int ar = anc ? anc[(long)row * ld_anc + lane] : row;
            ks = kcache + (long)lane * step_stride + (long)ar * ld_c + head * dk;
        }
        float s = 0.f;
        for (int c = 0; c < dk; ++c) s = fmaf(qr[c], ks[c], s);
        sc = s * scale;
        // teacher forcing masks key positions that hold pad/eos (except position 0), TransformerModel.py:324-328
        if (labels != nullptr && lane > 0 && labels[(long)row * ld_lab + lane] == 0) sc = -INFINITY;
    }
    const float mx = warp_max(sc);
    const float e = (lane <= t && sc > -INFINITY) ? expf(sc - mx) : 0.f;
    const float inv = 1.0f / warp_sum(e);
    // every lane runs every round, so the shuffles always see the whole warp: with a head narrower than 32 columns the lanes without a
    // column used to leave the loop, and the weights of positions >= the head width were read from exited lanes (undefined values)
    for (int c0 = 0; c0 < dk; c0 += 32) {
        const int c = c0 + lane;
        float acc = 0.f;
        for (int s = 0; s <= t; ++s) {
            const float w = __shfl_sync(0xffffffffu, e, s);
            if (c >= dk) continue;
            const float* vs;
            if (s == t) vs = vr;
            else {
                const int ar = anc ? anc[(long)row * ld_anc + s] : row;
                vs = vcache + (long)s * step_stride + (long)ar * ld_c + head * dk;
            }
            acc = fmaf(w, vs[c], acc);
        }
        if (c < dk) store_act2(out, row, head * dk + c, acc * inv);
    }
}

// The same attention at any step t (the positions past 31 that one lane per key cannot hold): one warp per (row, head) walks the positions
// 0..t in chunks of 32, one key per lane, with a running max and sum (online softmax).  Lane i owns output columns i, i + 32, ... (NC of them).
template <int NC>
__global__ void __launch_bounds__(128) dec_self_attention_long_kernel(int rows, int heads, int dk, int t, const float* __restrict__ qkv, long ld_qkv,
                                                                      float* __restrict__ kcache, float* __restrict__ vcache, long step_stride, long ld_c,
                                                                      const int* __restrict__ anc, long ld_anc, const long long* __restrict__ labels,
                                                                      long ld_lab, float scale, ActView out) {
    const int item = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (item >= rows * heads) return;
    const int lane = threadIdx.x & 31;
    const int row = item / heads, head = item % heads;
    const int D = heads * dk;
    const float* qr = qkv + (long)row * ld_qkv + head * dk;
    const float* kr = qr + D;
    const float* vr = qr + 2 * D;
    for (int c = lane; c < dk; c += 32) {
        kcache[(long)t * step_stride + (long)row * ld_c + head * dk + c] = kr[c];
        vcache[(long)t * step_stride + (long)row * ld_c + head * dk + c] = vr[c];
    }
    float m = -INFINITY, l = 0.f, acc[NC];
#pragma unroll
    for (int i = 0; i < NC; ++i) acc[i] = 0.f;
    for (int s0 = 0; s0 <= t; s0 += 32) {
        const int s = s0 + lane;
        const int ar = (s < t && anc != nullptr) ? anc[(long)row * ld_anc + s] : row;      // ancestor row holding position s
        float sc = -INFINITY;
        if (s <= t) {
            const float* ks = (s == t) ? kr : kcache + (long)s * step_stride + (long)ar * ld_c + head * dk;
            float d = 0.f;
            for (int c = 0; c < dk; ++c) d = fmaf(qr[c], ks[c], d);
            sc = d * scale;
            if (labels != nullptr && s > 0 && labels[(long)row * ld_lab + s] == 0) sc = -INFINITY;   // TransformerModel.py:324-328
        }
        const float m_new = fmaxf(m, warp_max(sc));
        if (m_new == -INFINITY) continue;                       // every position so far masked
        const float corr = expf(m - m_new);
        const float e = (sc > -INFINITY) ? expf(sc - m_new) : 0.f;
        l = l * corr + warp_sum(e);
        m = m_new;
#pragma unroll
        for (int i = 0; i < NC; ++i) acc[i] *= corr;
        const int n = (t + 1 - s0) < 32 ? (t + 1 - s0) : 32;
        for (int j = 0; j < n; ++j) {
            const float w = __shfl_sync(0xffffffffu, e, j);
            const int aj = __shfl_sync(0xffffffffu, ar, j);
            const float* vs = (s0 + j == t) ? vr : vcache + (long)(s0 + j) * step_stride + (long)aj * ld_c + head * dk;
#pragma unroll
            for (int i = 0; i < NC; ++i) {
                const int c = lane + 32 * i;
                if (c < dk) acc[i] = fmaf(w, vs[c], acc[i]);
            }
        }
    }
    const float inv = 1.0f / l;
#pragma unroll
    for (int i = 0; i < NC; ++i) {
        const int c = lane + 32 * i;
        if (c < dk) store_act2(out, row, head * dk + c, acc[i] * inv);
    }
}

// Single-query multi-head attention over per-image keys / values: one CTA per (row, head) (attn.cuh).
//   q [rows, ld_q]; kk, vv [B*R, ld_kv] (+ column offsets k_off / v_off); mask [B, R] or nullptr
__global__ void __launch_bounds__(128) cross_attention_kernel(int rows, int rpi, int heads, int dk, int R, const float* __restrict__ q, long ld_q,
                                                              const float* __restrict__ kk, const float* __restrict__ vv, long ld_kv,
                                                              const float* __restrict__ mask, long ld_mask, float scale, ActView out) {
    extern __shared__ float sm[];       // [R] scores -> exp
    __shared__ float sh_inv;
    const int item = blockIdx.x;
    const int row = item / heads, head = item % heads;
    const int img = row / rpi;
    const float* qr = q + (long)row * ld_q + head * dk;
    const float* kb = kk + (long)img * R * ld_kv + head * dk;
    const float* vb = vv + (long)img * R * ld_kv + head * dk;
    sq_attention_scores(qr, kb, ld_kv, R, dk, scale, mask != nullptr ? mask + (long)img * ld_mask : nullptr, sm);
    const float inv = sq_attention_softmax(sm, R, &sh_inv);
    for (int c = threadIdx.x; c < dk; c += 128) store_act2(out, row, head * dk + c, sq_attention_column(sm, vb, ld_kv, R, c) * inv);
}

// GLU over the last dimension (nn.GLU, AoAModel.py:41,143): out[r, j] = t[r, j] * sigmoid(t[r, H + j]) (+ residual[r, j])
__global__ void glu_kernel(int rows, int H, const float* __restrict__ t, long ld_t, const float* __restrict__ residual, long ld_res, ActView out) {
    const long total = (long)rows * H;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int r = (int)(i / H), j = (int)(i % H);
        const float a = t[(long)r * ld_t + j], b = t[(long)r * ld_t + H + j];
        float v = a * (1.0f / (1.0f + expf(-b)));
        if (residual != nullptr) v += residual[(long)r * ld_res + j];
        store_act2(out, r, j, v);
    }
}

// mean over the (valid) regions of each image (AoAModel.py:214-219): one CTA per image
__global__ void masked_mean_kernel(int R, int H, const float* __restrict__ x, long ld_x, const float* __restrict__ mask, long ld_mask, ActView out) {
    const int img = blockIdx.x;
    float cnt = 0.f;
    if (mask != nullptr) { for (int r = 0; r < R; ++r) cnt += mask[(long)img * ld_mask + r]; } else cnt = (float)R;
    for (int c = threadIdx.x; c < H; c += blockDim.x) {
        float s = 0.f;
        for (int r = 0; r < R; ++r) {
            const float v = x[((long)img * R + r) * ld_x + c];
            s += (mask != nullptr) ? v * mask[(long)img * ld_mask + r] : v;
        }
        store_act2(out, img, c, s / cnt);
    }
}

}  // namespace

int glu_launch(int rows, int H, const float* t, long ld_t, const float* residual, long ld_res, ActView out, cudaStream_t st) {
    if (rows <= 0) return 0;
    long blocks = ((long)rows * H + 255) / 256;
    if (blocks > sm_count() * 8) blocks = sm_count() * 8;
    glu_kernel<<<(int)blocks, 256, 0, st>>>(rows, H, t, ld_t, residual, ld_res, out);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int masked_mean_launch(int B, int R, int H, const float* x, long ld_x, const float* mask, long ld_mask, ActView out, cudaStream_t st) {
    if (B <= 0) return 0;
    masked_mean_kernel<<<B, 256, 0, st>>>(R, H, x, ld_x, mask, ld_mask, out);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int layer_norm_launch(int rows, int D, const float* x, long ld_x, const float* a, const float* b, float eps, ActView out, cudaStream_t st) {
    if (rows <= 0) return 0;
    layer_norm_kernel<<<rows, 128, 0, st>>>(rows, D, x, ld_x, a, b, eps, out);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int embed_pe_launch(int rows, int D, const int* tokens, const float* lut, const float* pe_row, float scale, ActView out, cudaStream_t st) {
    if (rows <= 0) return 0;
    embed_pe_kernel<<<rows, 128, 0, st>>>(rows, D, tokens, lut, pe_row, scale, out);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int enc_self_attention_launch(int B, int R, int heads, int dk, const float* q, const float* k, const float* v, long ld, const float* mask,
                              long ld_mask, ActView out, cudaStream_t st, int form) {
    if (B <= 0) return 0;
    const size_t smem = sizeof(float) * ((size_t)2 * R * (dk + 1) + 8 * R + 8 * dk);
    if (form == 2 || (form == 0 && smem > 200 * 1024))
        return attn_tiled_forward_launch(B, R, heads, dk, R, R, 1, q, k, v, ld, mask, ld_mask, 0ull, 0, 0.f, out, st);
    CAPB_REQUIRE(smem <= 200 * 1024, "self-attention: region count x head width too large for the shared-memory staging");
    int chunks = (296 + B * heads - 1) / (B * heads);           // query chunks: about two CTAs per SM even for a 10-image batch
    chunks = chunks > 4 ? 4 : (chunks < 1 ? 1 : chunks);
    if (chunks > R) chunks = R;
    static std::atomic<unsigned long long> configured{0};
    if (first_use_on_device(configured)) {
        CAPB_CHECK_CUDA(cudaFuncSetAttribute(enc_self_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    }
    enc_self_attention_kernel<<<dim3(B, heads, chunks), 256, smem, st>>>(R, dk, q, k, v, ld, mask, ld_mask, 1.0f / sqrtf((float)dk), out);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int dec_self_attention_launch(int rows, int heads, int dk, int t, const float* qkv, long ld_qkv, float* kcache, float* vcache, long step_stride,
                              long ld_c, const int* anc, long ld_anc, const long long* labels, long ld_lab, ActView out, cudaStream_t st, int form) {
    if (rows <= 0) return 0;
    CAPB_REQUIRE(t >= 0 && t <= CAPB200_MAX_SEQ_LENGTH, "decoder self-attention: position out of range (teacher forcing reaches seq_length)");
    const float scale = 1.0f / sqrtf((float)dk);
    if (form == 1 || (form == 0 && t < 32)) {
        CAPB_REQUIRE(t < 32, "decoder self-attention (one lane per position): handles up to 32 positions");
        dec_self_attention_kernel<<<cdiv(rows * heads, 4), 128, 0, st>>>(rows, heads, dk, t, qkv, ld_qkv, kcache, vcache, step_stride, ld_c, anc, ld_anc,
                                                                          labels, ld_lab, scale, out);
        CAPB_CHECK_CUDA(cudaGetLastError());
        return 0;
    }
    CAPB_REQUIRE(dk >= 1 && dk <= 256, "decoder self-attention: head width above 256");
    const int nc = dk <= 32 ? 1 : dk <= 64 ? 2 : dk <= 128 ? 4 : 8;
    const dim3 grid(cdiv(rows * heads, 4));
#define CAPB_DEC_LONG(N) dec_self_attention_long_kernel<N><<<grid, 128, 0, st>>>(rows, heads, dk, t, qkv, ld_qkv, kcache, vcache, step_stride, ld_c, anc, \
                                                                                 ld_anc, labels, ld_lab, scale, out)
    if (nc == 1) CAPB_DEC_LONG(1);
    else if (nc == 2) CAPB_DEC_LONG(2);
    else if (nc == 4) CAPB_DEC_LONG(4);
    else CAPB_DEC_LONG(8);
#undef CAPB_DEC_LONG
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int cross_attention_launch(int rows, int rpi, int heads, int dk, int R, const float* q, long ld_q, const float* kk, const float* vv, long ld_kv,
                           const float* mask, long ld_mask, ActView out, cudaStream_t st) {
    if (rows <= 0) return 0;
    const size_t smem = sizeof(float) * R;
    CAPB_REQUIRE(dk <= 256, "attention: head width above 256");
    cross_attention_kernel<<<rows * heads, 128, smem, st>>>(rows, rpi, heads, dk, R, q, ld_q, kk, vv, ld_kv, mask, ld_mask,
                                                                      1.0f / sqrtf((float)dk), out);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace capb200

extern "C" int capb200_tfm_dec_self_attention(int form, int rows, int heads, int dk, int t, const float* qkv, long ld_qkv, float* kcache, float* vcache,
                                              long step_stride, long ld_c, const int* anc, long ld_anc, const long long* labels, long ld_lab, float* out,
                                              long ld_out, void* stream) {
    CAPB_REQUIRE(form >= 0 && form <= 2, "form is 0 (automatic), 1 (one lane per position) or 2 (chunked)");
    CAPB_REQUIRE(rows > 0 && heads > 0 && dk > 0 && qkv && kcache && vcache && out, "bad argument");
    capb200::ActView o;
    o.f = out; o.ld = ld_out;
    return capb200::dec_self_attention_launch(rows, heads, dk, t, qkv, ld_qkv, kcache, vcache, step_stride, ld_c, anc, ld_anc, labels, ld_lab, o,
                                              static_cast<cudaStream_t>(stream), form);
}
