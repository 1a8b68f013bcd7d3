// Beam search's row statistics and top-k over one 16-byte aligned logit row, run by 128 threads: the body of vocab_stats_online128_kernel
// (vocab.cu, one CTA per row) and of each 128-thread group of beam_search_step_kernel (beam.cu, one CTA per image).  The reductions take
// a barrier functor, __syncthreads() for the whole CTA or a named barrier for one group, so both kernels compute the same bits.
#pragma once
#include "common.cuh"
#include "kernels.cuh"

namespace capb200 {

// Per-thread online softmax in base 2.  A thread's partial sum holds sum 2^(x*log2e - mL), where
// mL = fl(m*log2e) belongs to its running maximum m.  mL carries the rounding of that product -- up to half an ulp of |m|*log2e, 1e-4 at
// |m| = 1000 -- so the rescale to a new maximum and the final rescale to the row maximum are both taken against mL itself, not against m:
// the rounding then cancels and the log-sum-exp does not degrade with the magnitude of the logits (log_softmax is shift-invariant).
__device__ __forceinline__ void online_raise(float& part, float& m, float& mL, float m4) {
    const float nL = m4 * 1.4426950408889634f;
    float sc;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(sc) : "f"(mL - nL));
    part = (m == -INFINITY) ? 0.f : part * sc;      // a thread that has only seen -inf holds NaN (-inf - -inf), not a sum
    m = m4;
    mL = nL;
}
// the thread's share of sum exp(x - mx), mx = the row maximum
__device__ __forceinline__ float online_finish(float part, float m, float mL, float mx) {
    float sc;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(sc) : "f"(fmaf(-mx, 1.4426950408889634f, mL)));
    return (m == -INFINITY) ? 0.f : part * sc;
}

constexpr int VT2 = 128;

// barriers of the 128 threads that share a row: the whole CTA, or named barrier `id` (1..15) of one group
struct CtaBarrier {
    __device__ __forceinline__ void operator()() const { __syncthreads(); }
};
struct GroupBarrier {
    int id;
    __device__ __forceinline__ void operator()() const { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(VT2) : "memory"); }
};

// reductions over the 128 threads of a row (tid 0..127); scratch holds four entries
template <class Bar>
__device__ __forceinline__ float block_max4(float v, float* scratch, int tid, Bar bar) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    bar();
    if ((tid & 31) == 0) scratch[tid >> 5] = v;
    bar();
    return fmaxf(fmaxf(scratch[0], scratch[1]), fmaxf(scratch[2], scratch[3]));
}
template <class Bar>
__device__ __forceinline__ float block_sum4(float v, float* scratch, int tid, Bar bar) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    bar();
    if ((tid & 31) == 0) scratch[tid >> 5] = v;
    bar();
    return (scratch[0] + scratch[1]) + (scratch[2] + scratch[3]);
}
template <class Bar>
__device__ __forceinline__ void block_argmax4(float v, int i, float* sval, int* sidx, int tid, Bar bar, float& out_v, int& out_i) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, v, o);
        const int oi = __shfl_xor_sync(0xffffffffu, i, o);
        if (ov > v || (ov == v && oi < i)) { v = ov; i = oi; }
    }
    bar();
    if ((tid & 31) == 0) { sval[tid >> 5] = v; sidx[tid >> 5] = i; }
    bar();
    out_v = sval[0];
    out_i = sidx[0];
#pragma unroll
    for (int w = 1; w < VT2 / 32; ++w) {
        const float ov = sval[w];
        const int oi = sidx[w];
        if (ov > out_v || (ov == out_v && oi < out_i)) { out_v = ov; out_i = oi; }
    }
}

// Row r of a.logits: a.stats[r] = (max, log-sum-exp), and the a.topk best (log-prob, word) pairs, best first, to top_val / top_idx (row
// r's list, global or shared memory).  Per-thread online softmax (running max, partial sum rescaled when the max grows) and one
// max-of-four test in front of the top-2 bookkeeping, so the row is read once and the common path is ~5 instructions per element; four
// independent 128-bit loads in flight per thread.  Each thread sees only ~V1/512 float4s, so it keeps just its two best; the k arg-max
// rounds pop list heads and a thread whose list runs dry (it owned >= 3 of the top-k: rare) rescans its elements for the next one.
template <class Bar>
__device__ __forceinline__ void stats_online128_row(const VocabStepArgs& a, int r, int tid, Bar bar, float* s_red, int* s_idx, float* top_val,
                                                    int* top_idx) {
    const int n4 = a.V1 >> 2;
    const float4* g4 = reinterpret_cast<const float4*>(a.logits + (long)r * a.ld);
    constexpr float kL2E = 1.4426950408889634f;
    float t0v = -INFINITY, t1v = -INFINITY;
    int t0i = 0x7fffffff, t1i = 0x7fffffff;
    float m = -INFINITY, mL = -INFINITY, part = 0.f;
    auto consume = [&](const float4 x, int v) {
        const float m4 = fmaxf(fmaxf(x.x, x.y), fmaxf(x.z, x.w));
        if (m4 > m) {
            online_raise(part, m, mL, m4);
        }
        float e0, e1, e2, e3;
        asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e0) : "f"(fmaf(x.x, kL2E, -mL)));
        asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e1) : "f"(fmaf(x.y, kL2E, -mL)));
        asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e2) : "f"(fmaf(x.z, kL2E, -mL)));
        asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e3) : "f"(fmaf(x.w, kL2E, -mL)));
        part += (e0 + e1) + (e2 + e3);
        if (m4 > t1v) {                             // strict: earlier (lower) indices win ties
            const float xs[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                if (xs[u] > t1v) {
                    if (xs[u] > t0v) { t1v = t0v; t1i = t0i; t0v = xs[u]; t0i = 4 * v + u; }
                    else { t1v = xs[u]; t1i = 4 * v + u; }
                }
            }
        }
    };
    int v = tid;
    for (; v + 3 * VT2 < n4; v += 4 * VT2) {        // four loads in flight, consumed in index order (tie order is preserved)
        const float4 x0 = g4[v], x1 = g4[v + VT2], x2 = g4[v + 2 * VT2], x3 = g4[v + 3 * VT2];
        consume(x0, v); consume(x1, v + VT2); consume(x2, v + 2 * VT2); consume(x3, v + 3 * VT2);
    }
    for (; v < n4; v += VT2) consume(g4[v], v);
    const float mx = block_max4(m, s_red, tid, bar);
    float sum = online_finish(part, m, mL, mx);
    sum = block_sum4(sum, s_red, tid, bar);
    const float lsum = logf(sum);
    const float m2 = (mx - mx) - lsum, l2 = lsum;
    if (tid == 0) a.stats[r] = make_float2(mx, lsum);
    int popped = 0;
    for (int k = 0; k < a.topk; ++k) {
        float ov;
        int oi;
        block_argmax4(t0v, t0i, s_red, s_idx, tid, bar, ov, oi);
        if (t0i == oi && oi != 0x7fffffff) {
            const float lastv = t0v;
            const int lasti = t0i;
            t0v = t1v; t0i = t1i;
            t1v = -INFINITY; t1i = 0x7fffffff;
            if (++popped >= 2 && t0i == 0x7fffffff) {
                auto consider = [&](float x, int w) {
                    const bool after = (x < lastv) || (x == lastv && w > lasti);
                    if (after && (x > t0v || (x == t0v && w < t0i))) { t0v = x; t0i = w; }
                };
                for (int w = tid; w < n4; w += VT2) {
                    const float4 x = g4[w];
                    consider(x.x, 4 * w); consider(x.y, 4 * w + 1); consider(x.z, 4 * w + 2); consider(x.w, 4 * w + 3);
                }
            }
        }
        if (tid == 0) {
            const float lp = (ov - mx) - lsum;
            top_val[k] = a.row_twice(r) ? (lp - m2) - l2 : lp;
            top_idx[k] = oi;
        }
    }
}

}  // namespace capb200
