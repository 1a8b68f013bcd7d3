// Single-query attention of one (row, head) by one CTA of 128 threads (decode and train-mode forward share it).
//
// The rows are few (10 .. 1280) and every row-head pair is a chain of dependent global loads, so the kernel is built for loads in
// flight rather than for arithmetic: scores -- each warp takes chunks of eight regions and issues all of a chunk's key loads (lanes
// across the head's dk columns: coalesced 128-byte segments) before the first warp reduction; softmax -- warp 0; weighted sum --
// thread c owns column c and walks the regions twelve independent value loads at a time (one warp per pair with one dependent load
// per step was latency-bound).
#pragma once
#include <cuda_runtime.h>

namespace capb200 {

__device__ __forceinline__ float attn_wsum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float attn_wmax(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// scores p[r] = scale * q . K[r]  (-inf where mask_row[r] == 0); p in shared memory [R]; ends with __syncthreads()
__device__ __forceinline__ void sq_attention_scores(const float* __restrict__ qr, const float* __restrict__ kb, long ld_kv, int R, int dk, float scale,
                                                    const float* __restrict__ mask_row, float* __restrict__ p) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    constexpr int NQ = 8;               // dk <= 256
    float qv[NQ];
#pragma unroll
    for (int i = 0; i < NQ; ++i) { const int c = lane + 32 * i; qv[i] = (c < dk) ? qr[c] : 0.f; }
    for (int r0 = warp * 8; r0 < R; r0 += 32) {
        float part[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            part[u] = 0.f;
            if (r0 + u < R) {
                const float* kr = kb + (long)(r0 + u) * ld_kv;
#pragma unroll
                for (int i = 0; i < NQ; ++i) { const int c = lane + 32 * i; if (c < dk) part[u] = fmaf(qv[i], __ldg(kr + c), part[u]); }
            }
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            const float s = attn_wsum(part[u]) * scale;
            if (lane == 0 && r0 + u < R) p[r0 + u] = (mask_row != nullptr && mask_row[r0 + u] == 0.f) ? -INFINITY : s;
        }
    }
    __syncthreads();
}

// softmax over p[0..R) by warp 0 (in place: p[r] = exp(p[r] - max)); returns 1 / sum to every thread; ends with __syncthreads()
__device__ __forceinline__ float sq_attention_softmax(float* __restrict__ p, int R, float* __restrict__ sh_inv) {
    if (threadIdx.x < 32) {
        const int lane = threadIdx.x;
        float mx = -INFINITY;
        for (int r = lane; r < R; r += 32) mx = fmaxf(mx, p[r]);
        mx = attn_wmax(mx);
        float sum = 0.f;
        for (int r = lane; r < R; r += 32) { const float e = expf(p[r] - mx); p[r] = e; sum += e; }
        sum = attn_wsum(sum);
        if (lane == 0) *sh_inv = 1.0f / sum;
    }
    __syncthreads();
    return *sh_inv;
}

// acc = sum_r w[r] * V[r][c] for this thread's column c, twelve independent loads at a time
__device__ __forceinline__ float sq_attention_column(const float* __restrict__ w, const float* __restrict__ vb, long ld_kv, int R, int c) {
    float acc = 0.f;
    int r = 0;
    for (; r + 12 <= R; r += 12) {
        float v[12];
#pragma unroll
        for (int u = 0; u < 12; ++u) v[u] = __ldg(vb + (long)(r + u) * ld_kv + c);
#pragma unroll
        for (int u = 0; u < 12; ++u) acc = fmaf(w[r + u], v[u], acc);
    }
    for (; r < R; ++r) acc = fmaf(w[r], __ldg(vb + (long)r * ld_kv + c), acc);
    return acc;
}

}  // namespace capb200
