// Vocabulary epilogue: log-softmax (once for _sample, twice for beam search) and candidate selection.
//
// Replaces, per decode step:  F.log_softmax(self.logit(output))            AttModel.py:172
//                             F.log_softmax(logprobs / temperature)        CaptionModel.py:204   (beam search only; T = 1)
//                             torch.sort(b*(V+1) candidates)[:b]           CaptionModel.py:80-81 (per-row top-b, merged in beam.cu)
//                             torch.max / Categorical(logits).sample()     CaptionModel.py:372,405
//                             finished-row masking                         AttModel.py:340-347
// One CTA per row; the row lives in shared memory between the passes so HBM sees one read and one write.  Rows longer than one CTA's
// shared memory holds are spread over a thread-block cluster (vocab_step_cluster_kernel).
#include <cooperative_groups.h>
#include "common.cuh"
#include "kernels.cuh"
#include "vocab_row.cuh"

namespace cg = cooperative_groups;

namespace capb200 {

// seed salt of the sampling kernels (see dropout.cuh: lets a captured CUDA graph of the SCST step draw fresh samples on every replay)
static __device__ unsigned long long g_vocab_seed_salt = 0ull;
int dropout_salt_set_vocab(unsigned long long salt, cudaStream_t st) {
    return cudaMemcpyToSymbolAsync(g_vocab_seed_salt, &salt, sizeof(salt), 0, cudaMemcpyHostToDevice, st) == cudaSuccess ? 0 : 1;
}

namespace {

constexpr int VT = 256;   // threads per row

template <int NT = VT>
__device__ __forceinline__ float block_max(float v, float* scratch) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    __syncthreads();
    if ((threadIdx.x & 31) == 0) scratch[threadIdx.x >> 5] = v;
    __syncthreads();
    float r = scratch[0];
#pragma unroll
    for (int w = 1; w < NT / 32; ++w) r = fmaxf(r, scratch[w]);
    return r;
}

template <int NT = VT>
__device__ __forceinline__ float block_sum(float v, float* scratch) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) scratch[threadIdx.x >> 5] = v;
    __syncthreads();
    float r = 0.f;
#pragma unroll
    for (int w = 0; w < NT / 32; ++w) r += scratch[w];
    return r;
}

// arg-max with lowest-index tie-break; result broadcast to all threads
template <int NT = VT>
__device__ __forceinline__ void block_argmax(float v, int i, float* sval, int* sidx, float& out_v, int& out_i) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, v, o);
        const int oi = __shfl_xor_sync(0xffffffffu, i, o);
        if (ov > v || (ov == v && oi < i)) { v = ov; i = oi; }
    }
    __syncthreads();
    if ((threadIdx.x & 31) == 0) { sval[threadIdx.x >> 5] = v; sidx[threadIdx.x >> 5] = i; }
    __syncthreads();
    out_v = sval[0];
    out_i = sidx[0];
#pragma unroll
    for (int w = 1; w < NT / 32; ++w) {
        const float ov = sval[w];
        const int oi = sidx[w];
        if (ov > out_v || (ov == out_v && oi < out_i)) { out_v = ov; out_i = oi; }
    }
}

// Philox4x32-10 counter-based generator (Salmon et al. 2011): one 128-bit block per (element, row, step).
__device__ __forceinline__ uint32_t philox_first(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
    }
    return c0;
}

// The vocabulary step of row r for one CTA that caches the slice [red.lo, red.hi) of the row in `row`.  `red` supplies the row-wide
// reductions (RowInCta: block reductions; RowInCluster: block reductions followed by an exchange across the cluster), `red.lead` marks the
// CTA that writes the per-row outputs, and red.finish() is the barrier before they are written.
// Passes over the shared-memory copy of the row: (1) load + max, (2) sum exp, (3) log-probs + second-normalisation sum +
// per-thread sorted top-KMAX, (4) final values to HBM; then k arg-max rounds over the per-thread list heads.
// The second log_softmax only shifts the row by a constant, so candidates are ranked on the first-pass values.
template <int KMAX, int NT, class Red>
__device__ __forceinline__ void vocab_step_row(const VocabStepArgs& a, int r, float* row, Red& red) {
    const int lo = red.lo, hi = red.hi, n = hi - lo;
    float* g = a.logits + (long)r * a.ld + lo;

    if (a.unfinished != nullptr && !a.first_step && a.unfinished[r] == 0) {
        // sequence already ended: emit pad and a zero log-prob row (AttModel.py:342-344); every CTA of a cluster reads the same flag and
        // leaves here, touching no distributed shared memory
        for (int v = threadIdx.x; v < n; v += NT) g[v] = 0.f;
        if (red.lead && threadIdx.x == 0) {
            if (a.tokens_out) a.tokens_out[r] = 0;
            if (a.seq_out) a.seq_out[(long)r * a.ld_seq + a.t] = 0;
            if (a.picked_lp) a.picked_lp[(long)r * a.ld_picked] = 0.f;
        }
        return;
    }

    float mx = -INFINITY;
    for (int v = threadIdx.x; v < n; v += NT) { const float x = g[v]; row[v] = x; mx = fmaxf(mx, x); }
    mx = red.max(mx);
    float sum = 0.f;
    for (int v = threadIdx.x; v < n; v += NT) sum += __expf(row[v] - mx);
    sum = red.sum(sum);                          // ex2.approx path: relative error ~1e-7 on the sum
    const float lsum = logf(sum);
    const float m2 = (mx - mx) - lsum;            // max of the log-probs (second log_softmax)
    const int k_eff = a.topk > 0 ? a.topk : (a.select == 1 ? 1 : 0);
    float tv[KMAX];
    int ti[KMAX];
#pragma unroll
    for (int q = 0; q < KMAX; ++q) { tv[q] = -INFINITY; ti[q] = 0x7fffffff; }
    auto consider = [&](float lp, int v) {
        if (k_eff > 0 && lp > tv[KMAX - 1]) {
            float cv = lp;
            int ci = v;
#pragma unroll
            for (int q = 0; q < KMAX; ++q) {
                if (cv > tv[q]) { const float t0 = tv[q]; const int t1 = ti[q]; tv[q] = cv; ti[q] = ci; cv = t0; ci = t1; }
            }
        }
    };
    const bool edit = a.edits.any();
    for (int v = threadIdx.x; v < n; v += NT) {
        const float lp = (row[v] - mx) - lsum;
        row[v] = lp;
        if (!edit) consider(lp, lo + v);
    }
    if (edit) {
        // The reference's decode options edit the log-prob row AFTER the log-softmax, and the edited row is both what the next word is
        // chosen from and what is stored (AttModel.py:294-332).  A handful of columns change: one thread per CTA applies those of its
        // slice to the shared copy (a cluster repeats the trigram scan in every CTA: t^2 reads).
        __syncthreads();
        if (threadIdx.x == 0) {
            const int t = a.t;
            const int prev = (t > 0 && a.prev_tokens != nullptr) ? a.prev_tokens[r] : -1;
            if (a.edits.constraint && prev >= lo && prev < hi) row[prev - lo] = -INFINITY;             // never repeat the previous word
            bool prev_bad = false;
            for (int i = 0; i < a.edits.n_bad; ++i) prev_bad |= (t > 0 && a.edits.bad[i] == prev);
            if (prev_bad && red.lead) row[0] = -INFINITY;                                          // no end token after a bad ending
            if (a.edits.trigrams && t >= 3 && r < a.edits.trigram_rows && a.seq_out != nullptr) {
                const long long* sq = a.seq_out + (long)r * a.ld_seq;
                const long long p0 = sq[t - 2], p1 = sq[t - 1];
                for (int j = 0; j + 2 <= t - 1; ++j) {
                    if (sq[j] != p0 || sq[j + 1] != p1) continue;
                    const long long w = sq[j + 2];
                    bool first = true;
                    int count = 0;
                    for (int i = 0; i + 2 <= t - 1; ++i) {
                        if (sq[i] == p0 && sq[i + 1] == p1 && sq[i + 2] == w) { if (i < j) first = false; ++count; }
                    }
                    if (first && w >= lo && w < hi) row[w - lo] += ((float)count * -0.693f) * 2.0f;    // mask * -0.693 * alpha, alpha = 2 (AttModel.py:330-332)
                }
            }
        }
        __syncthreads();
        for (int v = threadIdx.x; v < n; v += NT) consider(row[v], lo + v);
    }
    // Second log_softmax (beam search, CaptionModel.py:204): its max is m2 = -lsum, so exp(lp - m2) = exp(x - mx) term by term and
    // its normaliser is the first pass's `sum` again (up to one rounding, ~1e-7 on the log-prob); no second exp pass is needed.
    const float l2 = lsum;
    if (a.row_twice(r)) {
        for (int v = threadIdx.x; v < n; v += NT) g[v] = (row[v] - m2) - l2;
    } else {
        for (int v = threadIdx.x; v < n; v += NT) g[v] = row[v];
    }

    int greedy_tok = 0;
    for (int k = 0; k < k_eff; ++k) {
        float ov;
        int oi;
        red.argmax(tv[0], ti[0], ov, oi);
        if (ti[0] == oi) {                        // the owner pops its head (column indices are global: one owner in the cluster)
#pragma unroll
            for (int q = 0; q + 1 < KMAX; ++q) { tv[q] = tv[q + 1]; ti[q] = ti[q + 1]; }
            tv[KMAX - 1] = -INFINITY;
            ti[KMAX - 1] = 0x7fffffff;
        }
        if (k == 0) greedy_tok = oi;
        if (a.topk > 0 && red.lead && threadIdx.x == 0) {
            a.top_val[(long)r * a.topk + k] = a.row_twice(r) ? (ov - m2) - l2 : ov;
            a.top_idx[(long)r * a.topk + k] = oi;
        }
    }

    int tok = 0;
    if (a.select == 3) {
        tok = a.forced[r];
    } else if (a.select == 1) {
        tok = greedy_tok;
    } else if (a.select != 0) {
        __syncthreads();
        const float inv_t = 1.0f / a.temperature;
        // order-preserving map float -> uint32 (for the threshold searches of the truncated samplers)
        auto okey = [](float x) { const uint32_t u = __float_as_uint(x); return (u & 0x80000000u) ? ~u : (u | 0x80000000u); };
        uint32_t keep_from = 0;                    // sample among the words whose key is >= keep_from
        if (a.select == 4) {
            // top-k (CaptionModel.py:398-402): threshold = k-th largest log-prob, by bisection on the key bits (exact; ties at the threshold are all kept)
            const float kf = floorf(a.top);
            for (int bit = 31; bit >= 0; --bit) {
                const uint32_t cand = keep_from | (1u << bit);
                float cnt = 0.f;
                for (int v = threadIdx.x; v < n; v += NT) cnt += (okey(row[v]) >= cand) ? 1.f : 0.f;
                cnt = red.sum(cnt);        // exact: counts stay below 2^24
                if (cnt >= kf) keep_from = cand;
            }
        } else if (a.select == 5) {
            // nucleus (CaptionModel.py:388-397): a word is kept iff the probability mass of the strictly more likely words is < p
            float mxl = -INFINITY;
            for (int v = threadIdx.x; v < n; v += NT) mxl = fmaxf(mxl, row[v]);
            mxl = red.max(mxl);
            float z = 0.f;
            for (int v = threadIdx.x; v < n; v += NT) z += __expf((row[v] - mxl) * inv_t);
            z = red.sum(z);
            const float target = a.top * z;
            auto mass_above = [&](uint32_t key) {   // sum over the words with key > `key`
                float m = 0.f;
                for (int v = threadIdx.x; v < n; v += NT) m += (okey(row[v]) > key) ? __expf((row[v] - mxl) * inv_t) : 0.f;
                return red.sum(m);
            };
            // largest key F with mass_above(F) >= target; everything above F is kept (the most likely word always is)
            uint32_t F = 0;
            if (mass_above(0u) < target) keep_from = 0;
            else {
                for (int bit = 31; bit >= 0; --bit) {
                    const uint32_t cand = F | (1u << bit);
                    if (mass_above(cand) >= target) F = cand;
                }
                keep_from = F + 1u;
            }
        }
        float bv = -INFINITY;
        int bi = 0x7fffffff;
        const unsigned long long sd = a.seed ^ g_vocab_seed_salt;           // see dropout.cuh: graph replays of the SCST step
        const uint32_t k0 = (uint32_t)sd, k1 = (uint32_t)(sd >> 32);
        for (int v = threadIdx.x; v < n; v += NT) {
            if (okey(row[v]) < keep_from) continue;
            const int w = lo + v;
            const uint32_t bits = philox_first((uint32_t)w, (uint32_t)r, (uint32_t)a.step, (uint32_t)(a.step >> 32), k0, k1);
            const float u = ((float)(bits >> 9) + 0.5f) * (1.0f / 8388608.0f);      // (0,1), 23 bits
            const float x = row[v] * inv_t - logf(-logf(u));                         // Gumbel-max sample of softmax(logp / T)
            if (x > bv) { bv = x; bi = w; }
        }
        float ov;
        red.argmax(bv, bi, ov, tok);
    }
    // After this barrier every thread (every CTA of a cluster) has read unfinished[r] and prev_tokens[r] (tokens_out may alias
    // prev_tokens) before the lead CTA rewrites them, and no CTA of a cluster reads another's slots any more (so any may leave).
    red.finish();
    if (a.select != 0 && threadIdx.x == 0) {
        if (red.lead) {
            if (a.unfinished) a.unfinished[r] = (tok != 0) ? 1 : 0;
            if (a.tokens_out) a.tokens_out[r] = tok;
            if (a.seq_out) a.seq_out[(long)r * a.ld_seq + a.t] = tok;
        }
        if (a.picked_lp && tok >= lo && tok < hi) a.picked_lp[(long)r * a.ld_picked] = row[tok - lo];
    }
}

template <int NT>
struct RowInCta {
    float* s_red;
    int* s_idx;
    int lo, hi;
    bool lead;
    __device__ float max(float v) { return block_max<NT>(v, s_red); }
    __device__ float sum(float v) { return block_sum<NT>(v, s_red); }
    __device__ void argmax(float v, int i, float& ov, int& oi) { block_argmax<NT>(v, i, s_red, s_idx, ov, oi); }
    __device__ void finish() { __syncthreads(); }
};

// One CTA per row, the whole row in shared memory (V1 <= kRowSmem).
// NT threads per row: 256 in general; 1024 for the few-row sampling / greedy steps of the training loops, where one CTA per row leaves the
// machine nearly empty and the row passes (37 elements per thread at 256 threads, a Philox draw each) are the whole cost
template <int KMAX, int NT = VT>
__global__ void __launch_bounds__(NT) vocab_step_kernel(const VocabStepArgs a) {
    extern __shared__ float row[];                // [V1]
    __shared__ float s_red[NT / 32];
    __shared__ int s_idx[NT / 32];
    RowInCta<NT> red{s_red, s_idx, 0, a.V1, true};
    vocab_step_row<KMAX, NT>(a, blockIdx.x, row, red);
}

// ---- Rows of more than kRowSmem entries: the same step on a thread-block cluster ------------------------------------------------
// One row per cluster of C = ceil(V1 / kRowSmem) CTAs (C <= 8, the portable cluster size): CTA c caches the slice [c*S, min(V1, (c+1)*S)),
// S = ceil(V1 / C), in its shared memory, so the row still crosses HBM once each way however many passes the samplers make over it.
// Every block-wide reduction of vocab_step_kernel is followed by a reduction across the cluster through distributed shared memory.
constexpr int kRowSmem = 51200;                  // floats of one row a CTA caches: 200 KB
constexpr int kMaxCluster = 8;
constexpr int kMaxRow = kRowSmem * kMaxCluster;  // 409 600
constexpr int VTC = 512;                         // threads per CTA of the cluster form, chosen by measurement (DESIGN.md)

// Each CTA publishes its block result in a slot of its own shared memory; after one cluster barrier the first C threads fetch the C
// slots and every thread combines them in rank order, so all CTAs of the cluster hold the same bits.  The slots alternate between two
// parities: a slot is rewritten two reductions later, after the barrier that every reader passes only once it has read it.
struct ClusterSlots {
    float v[2];
    int i[2];
    float gv[kMaxCluster];
    int gi[kMaxCluster];
};

__device__ __forceinline__ void cluster_exchange(float v, int i, ClusterSlots& cs, int& par) {
    cg::cluster_group cl = cg::this_cluster();
    if (threadIdx.x == 0) { cs.v[par] = v; cs.i[par] = i; }
    cl.sync();                                   // barrier.cluster.arrive.release + wait.acquire: the slots are visible
    if (threadIdx.x < cl.num_blocks()) {
        const ClusterSlots* rs = cl.map_shared_rank(&cs, threadIdx.x);
        cs.gv[threadIdx.x] = rs->v[par];
        cs.gi[threadIdx.x] = rs->i[par];
    }
    __syncthreads();
    par ^= 1;
}

template <int NT>
__device__ __forceinline__ float cluster_max(float v, float* s_red, ClusterSlots& cs, int& par) {
    cluster_exchange(block_max<NT>(v, s_red), 0, cs, par);
    const int C = (int)cg::this_cluster().num_blocks();
    float r = cs.gv[0];
    for (int c = 1; c < C; ++c) r = fmaxf(r, cs.gv[c]);
    return r;
}

template <int NT>
__device__ __forceinline__ float cluster_sum(float v, float* s_red, ClusterSlots& cs, int& par) {
    cluster_exchange(block_sum<NT>(v, s_red), 0, cs, par);
    const int C = (int)cg::this_cluster().num_blocks();
    float r = cs.gv[0];
    for (int c = 1; c < C; ++c) r += cs.gv[c];
    return r;
}

// arg-max with lowest-index tie-break over the whole row
template <int NT>
__device__ __forceinline__ void cluster_argmax(float v, int i, float* s_red, int* s_idx, ClusterSlots& cs, int& par, float& out_v, int& out_i) {
    float bv;
    int bi;
    block_argmax<NT>(v, i, s_red, s_idx, bv, bi);
    cluster_exchange(bv, bi, cs, par);
    const int C = (int)cg::this_cluster().num_blocks();
    out_v = cs.gv[0];
    out_i = cs.gi[0];
    for (int c = 1; c < C; ++c) {
        if (cs.gv[c] > out_v || (cs.gv[c] == out_v && cs.gi[c] < out_i)) { out_v = cs.gv[c]; out_i = cs.gi[c]; }
    }
}

template <int NT>
struct RowInCluster {
    float* s_red;
    int* s_idx;
    ClusterSlots* cs;
    int par;
    int lo, hi;
    bool lead;
    __device__ float max(float v) { return cluster_max<NT>(v, s_red, *cs, par); }
    __device__ float sum(float v) { return cluster_sum<NT>(v, s_red, *cs, par); }
    __device__ void argmax(float v, int i, float& ov, int& oi) { cluster_argmax<NT>(v, i, s_red, s_idx, *cs, par, ov, oi); }
    __device__ void finish() { cg::this_cluster().sync(); }
};

// vocab_step_kernel with the row split over a cluster (rows of 51 201 .. 409 600 entries).  Same passes, same tie order, same Philox
// block per (word, row, step, seed): the drawn word does not depend on how the row is split.  The row's sum is combined in rank order,
// so its log-probs may differ from what one CTA would compute in the last bit; there is no one-CTA form at these lengths.
template <int KMAX, int NT>
__global__ void __launch_bounds__(NT) vocab_step_cluster_kernel(const VocabStepArgs a, int S) {
    extern __shared__ float row[];               // [S]: this CTA's slice of the row
    __shared__ float s_red[NT / 32];
    __shared__ int s_idx[NT / 32];
    __shared__ ClusterSlots cs;
    cg::cluster_group cl = cg::this_cluster();
    const int rank = (int)cl.block_rank();
    const int lo = rank * S;
    RowInCluster<NT> red{s_red, s_idx, &cs, 0, lo, min(a.V1, lo + S), rank == 0};
    vocab_step_row<KMAX, NT>(a, blockIdx.x / cl.num_blocks(), row, red);
}

// Beam-search variant: the raw logits stay where the GEMM wrote them (they are normalised lazily, only for the rows that end up in
// the output); this kernel streams each row twice from L2 (max, then sum-exp + per-thread top-k) and writes only the row statistics
// and the top-k candidates.  Halves the HBM traffic of the step's vocabulary epilogue.
// Each thread sees only ~V1/256 elements, so it keeps just its two best; the k block-wide arg-max rounds pop list heads and a
// thread whose list runs dry (it owned >= 3 of the global top-k: rare) rescans its elements for the next one.
__global__ void __launch_bounds__(VT) vocab_stats_kernel(const VocabStepArgs a) {
    __shared__ float s_red[VT / 32];
    __shared__ int s_idx[VT / 32];
    const int r = blockIdx.x;
    const int V1 = a.V1;
    const float* g = a.logits + (long)r * a.ld;
    const bool vec = ((V1 & 3) == 0) && ((a.ld & 3) == 0) && ((reinterpret_cast<uintptr_t>(a.logits) & 15) == 0);
    float mx = -INFINITY;
    if (vec) {
        const float4* g4 = reinterpret_cast<const float4*>(g);
        for (int v = threadIdx.x; v < V1 / 4; v += VT) { const float4 x = g4[v]; mx = fmaxf(mx, fmaxf(fmaxf(x.x, x.y), fmaxf(x.z, x.w))); }
    } else {
        for (int v = threadIdx.x; v < V1; v += VT) mx = fmaxf(mx, g[v]);
    }
    mx = block_max(mx, s_red);
    float t0v = -INFINITY, t1v = -INFINITY;
    int t0i = 0x7fffffff, t1i = 0x7fffffff;
    float sum = 0.f;
    auto visit = [&](float x, int v) {
        sum += __expf(x - mx);
        if (x > t1v) {                              // strict: earlier (lower) indices win ties
            if (x > t0v) { t1v = t0v; t1i = t0i; t0v = x; t0i = v; }
            else { t1v = x; t1i = v; }
        }
    };
    if (vec) {
        const float4* g4 = reinterpret_cast<const float4*>(g);
        for (int v = threadIdx.x; v < V1 / 4; v += VT) {
            const float4 x = g4[v];
            visit(x.x, 4 * v); visit(x.y, 4 * v + 1); visit(x.z, 4 * v + 2); visit(x.w, 4 * v + 3);
        }
    } else {
        for (int v = threadIdx.x; v < V1; v += VT) visit(g[v], v);
    }
    sum = block_sum(sum, s_red);
    const float lsum = logf(sum);
    const float m2 = (mx - mx) - lsum, l2 = lsum;
    if (threadIdx.x == 0) a.stats[r] = make_float2(mx, lsum);
    int popped = 0;
    for (int k = 0; k < a.topk; ++k) {
        float ov;
        int oi;
        block_argmax(t0v, t0i, s_red, s_idx, ov, oi);
        if (t0i == oi && oi != 0x7fffffff) {
            const float lastv = t0v;
            const int lasti = t0i;
            t0v = t1v; t0i = t1i;
            t1v = -INFINITY; t1i = 0x7fffffff;
            if (++popped >= 2 && t0i == 0x7fffffff) {
                // rescan my elements for the best one ordered after (lastv, lasti)
                auto consider = [&](float x, int v) {
                    const bool after = (x < lastv) || (x == lastv && v > lasti);
                    if (after && (x > t0v || (x == t0v && v < t0i))) { t0v = x; t0i = v; }
                };
                if (vec) {
                    const float4* g4 = reinterpret_cast<const float4*>(g);
                    for (int v = threadIdx.x; v < V1 / 4; v += VT) {
                        const float4 x = g4[v];
                        consider(x.x, 4 * v); consider(x.y, 4 * v + 1); consider(x.z, 4 * v + 2); consider(x.w, 4 * v + 3);
                    }
                } else {
                    for (int v = threadIdx.x; v < V1; v += VT) consider(g[v], v);
                }
            }
        }
        if (threadIdx.x == 0) {
            const float lp = (ov - mx) - lsum;
            a.top_val[(long)r * a.topk + k] = a.row_twice(r) ? (lp - m2) - l2 : lp;
            a.top_idx[(long)r * a.topk + k] = oi;
        }
    }
}

// Single-pass variant of vocab_stats_kernel for 16-byte aligned rows (stats_online128_row, vocab_row.cuh).  128 threads: 16 CTAs per SM
// (all 1280 rows of the headline shape resident at once, no tail wave) and four independent 128-bit loads in flight per thread.
__global__ void __launch_bounds__(VT2) vocab_stats_online128_kernel(const VocabStepArgs a) {
    __shared__ float s_red[VT2 / 32];
    __shared__ int s_idx[VT2 / 32];
    const int r = blockIdx.x;
    stats_online128_row(a, r, threadIdx.x, CtaBarrier{}, s_red, s_idx, a.top_val + (long)r * a.topk, a.top_idx + (long)r * a.topk);
}

// Scheduled sampling (AttModel.py:145-154): with probability `prob` the word fed into step `col` is drawn from the model's own previous
// prediction exp(logprobs[:, col-1]) instead of the label.  One CTA per row; per-row uniform and the Gumbel-max draw come from the Philox
// stream (seed, site 6, step col).  Non-differentiable by construction (the reference samples from a detached tensor).
__global__ void __launch_bounds__(VT) ss_select_kernel(int V1, const float* __restrict__ prev_logp, long ld, const long long* __restrict__ labels,
                                                      long ld_labels, int col, unsigned long long seed, float prob, int* __restrict__ tok_out) {
    __shared__ float s_red[VT / 32];
    __shared__ int s_idx[VT / 32];
    const int r = blockIdx.x;
    seed ^= g_vocab_seed_salt;
    const uint32_t k0 = (uint32_t)seed ^ 0x6a09e667u, k1 = (uint32_t)(seed >> 32) ^ 0xbb67ae85u;
    const uint32_t ubits = philox_first(0xffffffffu, (uint32_t)r, (uint32_t)col, 6u, k0, k1);
    const float u_row = ((float)(ubits >> 9) + 0.5f) * (1.0f / 8388608.0f);
    if (!(u_row < prob)) {                       // keep the label (uniform over the whole CTA: no divergence at the barriers below)
        if (threadIdx.x == 0) tok_out[r] = (int)labels[(long)r * ld_labels + col];
        return;
    }
    const float* g = prev_logp + (long)r * ld;
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int v = threadIdx.x; v < V1; v += VT) {
        const uint32_t bits = philox_first((uint32_t)v, (uint32_t)r, (uint32_t)col, 6u, k0, k1);
        const float u = ((float)(bits >> 9) + 0.5f) * (1.0f / 8388608.0f);
        const float x = g[v] - logf(-logf(u));                  // Gumbel-max draw from softmax(logp) = exp(logp)
        if (x > bv) { bv = x; bi = v; }
    }
    float ov;
    int tok;
    block_argmax(bv, bi, s_red, s_idx, ov, tok);
    if (threadIdx.x == 0) tok_out[r] = tok;
}

__global__ void mask_rows_kernel(ActView x, int R, int cols, const float* __restrict__ mask, long ld_mask) {
    const int row = blockIdx.x;              // row = img * R + r
    const int img = row / R, r = row % R;
    if (mask[(long)img * ld_mask + r] != 0.f) return;
    for (int c = threadIdx.x; c < cols; c += blockDim.x) {
        x.f[(long)row * x.ld + c] = 0.f;
        if (x.hi) { x.hi[(long)row * x.ld + c] = __float2half(0.f); x.lo[(long)row * x.ld + c] = __float2half(0.f); }
    }
}

template <int KMAX>
int vocab_step_cluster_launch_k(const VocabStepArgs& a, cudaStream_t stream) {
    const int C = cdiv(a.V1, kRowSmem);
    const int S = cdiv(a.V1, C);
    static std::atomic<unsigned long long> configured{0};
    if (first_use_on_device(configured)) {
        CAPB_CHECK_CUDA(cudaFuncSetAttribute(vocab_step_cluster_kernel<KMAX, VTC>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)(sizeof(float) * kRowSmem)));
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(a.rows * C));
    cfg.blockDim = dim3(VTC);
    cfg.dynamicSmemBytes = sizeof(float) * (size_t)S;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)C;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    CAPB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, vocab_step_cluster_kernel<KMAX, VTC>, a, S));
    return 0;
}

int vocab_step_cluster_launch(const VocabStepArgs& a, cudaStream_t stream) {
    if (a.topk <= 2) return vocab_step_cluster_launch_k<2>(a, stream);
    if (a.topk <= 8) return vocab_step_cluster_launch_k<8>(a, stream);
    return vocab_step_cluster_launch_k<16>(a, stream);
}

}  // namespace

int vocab_step_launch(const VocabStepArgs& a, cudaStream_t stream) {
    if (a.rows <= 0) return 0;
    CAPB_REQUIRE(a.topk <= 16, "beam size up to 16");
    if (a.stats != nullptr) {
        CAPB_REQUIRE(a.select == 0 && a.topk > 0, "stats mode is the beam-search epilogue");
        const bool vec = ((a.V1 & 3) == 0) && ((a.ld & 3) == 0) && ((reinterpret_cast<uintptr_t>(a.logits) & 15) == 0);
        if (vec) vocab_stats_online128_kernel<<<a.rows, VT2, 0, stream>>>(a);
        else vocab_stats_kernel<<<a.rows, VT, 0, stream>>>(a);        // scalar loads: misaligned rows or V1 not a multiple of 4
        CAPB_CHECK_CUDA(cudaGetLastError());
        return 0;
    }
    CAPB_REQUIRE(a.V1 <= kMaxRow, "the vocabulary step supports up to 409600 entries per row (V + 1 <= 409600, a cluster of 8 CTAs "
                                  "caching 51200 entries each)");
    if (a.V1 > kRowSmem) return vocab_step_cluster_launch(a, stream);
    const size_t smem = sizeof(float) * (size_t)a.V1;
    static std::atomic<unsigned long long> configured{0};
    if (first_use_on_device(configured)) {
        CAPB_CHECK_CUDA(cudaFuncSetAttribute(vocab_step_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(200 * 1024)));
        CAPB_CHECK_CUDA(cudaFuncSetAttribute(vocab_step_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(200 * 1024)));
        CAPB_CHECK_CUDA(cudaFuncSetAttribute(vocab_step_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(200 * 1024)));
    }
    if (a.topk <= 2 && a.select != 0 && a.rows <= 2 * sm_count()) {
        static std::atomic<unsigned long long> configured2{0};
        if (first_use_on_device(configured2)) {
            CAPB_CHECK_CUDA(cudaFuncSetAttribute(vocab_step_kernel<2, 1024>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(200 * 1024)));
        }
        vocab_step_kernel<2, 1024><<<a.rows, 1024, smem, stream>>>(a);
    }
    else if (a.topk <= 2) vocab_step_kernel<2><<<a.rows, VT, smem, stream>>>(a);
    else if (a.topk <= 8) vocab_step_kernel<8><<<a.rows, VT, smem, stream>>>(a);
    else vocab_step_kernel<16><<<a.rows, VT, smem, stream>>>(a);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int ss_select_launch(int rows, int V1, const float* prev_logp, long ld, const long long* labels, long ld_labels, int col, unsigned long long seed, float prob,
                     int* tok_out, cudaStream_t stream) {
    if (rows <= 0) return 0;
    ss_select_kernel<<<rows, VT, 0, stream>>>(V1, prev_logp, ld, labels, ld_labels, col, seed, prob, tok_out);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int mask_rows_launch(ActView x, int n_images, int R, int cols, const float* mask, long ld_mask, cudaStream_t stream) {
    if (n_images <= 0 || mask == nullptr) return 0;
    mask_rows_kernel<<<n_images * R, 128, 0, stream>>>(x, R, cols, mask, ld_mask);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace capb200
