// Device-resident beam search bookkeeping (CaptionModel.beam_search: the group_size == 1 path and diverse beam search).
//
// The reference (captioning/models/CaptionModel.py:60-110,148-207) sorts all b*(V+1) candidates per image, gathers and
// re-concatenates the whole [B,b,t,V+1] log-prob history every step, runs three .all() host syncs and a Python loop with
// .item() per finished beam.  Here hypotheses stay on the device for all T steps:
//   * vocab.cu leaves the per-row top-b (value, word) pairs; beam_step merges live*b candidates per image in registers,
//   * token / slab-row histories are b*T ints per image, reordered by parent pointer,
//   * finished beams are appended to a per-image record list (<= b*T entries), exactly mirroring the reference's
//     quirks: a beam that emits EOS (or any beam at the last step) is recorded with its current sum, then its running sum
//     is lowered by 1000 but it stays in the beam and keeps being expanded (CaptionModel.py:183-198),
//   * the full log-prob rows are never copied while searching: each step's [rows, V+1] slab stays where the vocab kernel
//     wrote it and the winner's rows are gathered once at the end (AttModel.py:245-254 semantics).
#include "../../include/capb200.h"
#include "common.cuh"
#include "kernels.cuh"
#include "vocab_row.cuh"

namespace capb200 {

namespace {

constexpr int MAXB = 16;

__device__ __forceinline__ double apply_penalty(int kind, float alpha, int length, double p) {
    if (kind == 1) return p / (pow(5.0 + length, (double)alpha) / pow(6.0, (double)alpha));   // 'wu_<alpha>'  misc.py:137-145
    if (kind == 2) return p / (double)length;                                                  // 'avg_<alpha>' misc.py:147-151
    return p;
}

// One step of the search for one image (or one group of an image in diverse beam search), run by one warp.  `img` indexes the sums /
// sequence tables / records (s.beam beams each); the `live` parent rows of this step are rows row0 .. row0 + live - 1, whose `kl`
// candidates each are top_val / top_idx[(row - row0) * kl + k] (global memory, or shared memory in beam_search_step_kernel).  The n_pen
// words at `pen` (shared memory) lower a candidate by lambda per occurrence (add_diversity,
// CaptionModel.py:38-55).  Chosen words go to s.tokens / s.src_row[img * beam + j] with parent row row0 + parent; the log-prob slab row
// of a record is hist0 + parent.  Each lane holds U candidates (lane, lane + 32, ...): live * kl <= 32 * U.  Slots past the candidates
// never win, so U does not change the result.
template <int U = 8>
__device__ __forceinline__ void select_step(const BeamState& s, int img, int t, int live, int kl, int row0, int hist0, const float* top_val,
                                            const int* top_idx, const int* pen, int n_pen, float lambda, int penalty_kind,
                                            float penalty_alpha, double* __restrict__ done_p) {
    const int lane = threadIdx.x;
    const int b = s.beam, T = s.T;
    const int ncand = live * kl;
    // each lane owns candidates lane, lane+32, ... (ncand <= 32 * U)
    float cv[U];
    int cf[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
        const int c = lane + 32 * u;
        cv[u] = -INFINITY;
        cf[u] = 0x7fffffff;
        if (c < ncand) {
            const int pb = c / kl, k = c % kl;
            const int w = top_idx[pb * kl + k];
            float v = top_val[pb * kl + k];
            int cnt = 0;
            for (int q = 0; q < n_pen; ++q) cnt += (pen[q] == w);
            if (cnt) v = __fsub_rn(v, __fmul_rn((float)cnt, lambda));     // logprobs - change * diversity_lambda
            cv[u] = s.sums[(long)img * b + pb] + v;                          // same fp32 add as CaptionModel.py:79
            cf[u] = pb * s.V1 + w;                                           // flat index into the [live*(V+1)] candidate list
        }
    }

    const int* seq_old = (t & 1) ? s.seq_b : s.seq_a;
    int* seq_new = (t & 1) ? s.seq_a : s.seq_b;
    const int* hist_old = (t & 1) ? s.hist_b : s.hist_a;
    int* hist_new = (t & 1) ? s.hist_a : s.hist_b;

    // ---- phase 1: the b winners in order (registers and shuffles only); lane j keeps winner j
    float my_v = -INFINITY;
    int my_f = 0;
    for (int j = 0; j < b; ++j) {
        // arg-max over the remaining candidates; ties -> lowest flat index
        float bv = -INFINITY;
        int bf = 0x7fffffff, bu = -1;
#pragma unroll
        for (int u = 0; u < U; ++u)
            if (cv[u] > bv || (cv[u] == bv && cf[u] < bf)) { bv = cv[u]; bf = cf[u]; bu = u; }
        float wv = bv;
        int wf = bf;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, wv, o);
            const int of = __shfl_xor_sync(0xffffffffu, wf, o);
            if (ov > wv || (ov == wv && of < wf)) { wv = ov; wf = of; }
        }
        if (bu >= 0 && bf == wf && bv == wv) {       // the owning lane retires the winner
#pragma unroll
            for (int u = 0; u < U; ++u) if (u == bu) { cv[u] = -INFINITY; cf[u] = 0x7fffffff; }
        }
        if (lane == j) { my_v = wv; my_f = wf; }
    }
    // ---- phase 2: all history copies in parallel (the serial per-winner version was a chain of dependent global round trips)
    __shared__ int sh_parent[MAXB], sh_word[MAXB], sh_slot[MAXB];
    const bool has = lane < b;
    const int parent = has ? my_f / s.V1 : 0;
    const int word = has ? my_f % s.V1 : 0;
    const bool ended = has && ((word == 0) || (t == T - 1));
    const unsigned em = __ballot_sync(0xffffffffu, ended);
    const int cnt0 = s.done_cnt[img];
    const int slot = cnt0 + __popc(em & ((1u << lane) - 1u));          // records are appended in winner order
    if (has) { sh_parent[lane] = parent; sh_word[lane] = word; sh_slot[lane] = ended ? slot : -1; }
    __syncwarp();
#pragma unroll 1      // not unrolled: the 48-register beam_search_step_kernel holds this loop without spills
    for (int idx = lane; idx < b * t; idx += 32) {
        const int j = idx / t, q = idx - j * t;
        const long dst = ((long)img * b + j) * T, src = ((long)img * b + sh_parent[j]) * T;
        seq_new[dst + q] = seq_old[src + q];
        hist_new[dst + q] = hist_old[src + q];
    }
    if (em != 0u) {
#pragma unroll 1
        for (int idx = lane; idx < b * (t + 1); idx += 32) {
            const int j = idx / (t + 1), q = idx - j * (t + 1);
            if (sh_slot[j] < 0) continue;
            const long rec = ((long)img * b * T + sh_slot[j]) * T, src = ((long)img * b + sh_parent[j]) * T;
            s.done_seq[rec + q] = (q < t) ? seq_old[src + q] : sh_word[j];
            s.done_hist[rec + q] = (q < t) ? hist_old[src + q] : hist0 + sh_parent[j];
        }
    }
    if (has) {
        const long dst = ((long)img * b + lane) * T;
        seq_new[dst + t] = word;
        hist_new[dst + t] = hist0 + parent;
        float new_sum = my_v;
        if (ended) {
            const long rec = (long)img * b * T + slot;
            s.done_len[rec] = t + 1;
            s.done_raw[rec] = new_sum;
            done_p[rec] = apply_penalty(penalty_kind, penalty_alpha, t + 1, (double)new_sum);
            new_sum -= 1000.0f;
        }
        s.sums[(long)img * b + lane] = new_sum;
        s.tokens[(long)img * b + lane] = word;
        s.src_row[(long)img * b + lane] = row0 + parent;
    }
    if (lane == 0 && em != 0u) s.done_cnt[img] = cnt0 + __popc(em);
}

// one warp per image
__global__ void __launch_bounds__(32) beam_step_kernel(BeamState s, int t, int live, const float* __restrict__ top_val,
                                                       const int* __restrict__ top_idx, int penalty_kind, float penalty_alpha,
                                                       double* __restrict__ done_p) {
    const int img = blockIdx.x;
    const long row0 = (long)img * live;
    select_step(s, img, t, live, s.beam, (int)row0, (int)row0, top_val + row0 * s.beam, top_idx + row0 * s.beam, nullptr, 0, 0.f, penalty_kind,
                penalty_alpha, done_p);
}

// One CTA per image: vocab_stats_online128_kernel over the image's `live` rows, beam_step_kernel, and (t < T - 1) the parent-state gather
// of state_gather_embed_kernel for the next step, in one launch.  Rows are image-major and a row's parent is a row of the same image, so
// nothing crosses CTAs.  min(live, 8) groups of 128 threads; group g takes rows g, g + 8, ... and runs exactly the per-row work of
// vocab_stats_online128_kernel (same partition and reduction order, named barrier 1 + g for its reductions), so the row statistics and
// the top lists are bitwise those of the separate kernels; the top lists stay in shared memory.  U = 2 (beam <= 8, at most 64 candidates)
// fits 48 registers: two CTAs of 640 threads (beam 5) per SM, so the 256 images of the headline shape are resident in one wave on 132 SMs.
// U = 8 (beam 9..16) runs 1024 threads, one CTA per SM, and gets 64.
constexpr int kStepGroups = 8;
template <int U>
__global__ void __maxnreg__(U <= 2 ? 48 : 64) beam_search_step_kernel(BeamState s, const VocabStepArgs a, int t, int live, int penalty_kind, float penalty_alpha,
                                                        double* __restrict__ done_p, NextStateGather next) {
    __shared__ float s_red[kStepGroups][VT2 / 32];
    __shared__ int s_ridx[kStepGroups][VT2 / 32];
    __shared__ float s_val[MAXB * MAXB];
    __shared__ int s_idx[MAXB * MAXB];
    const int img = blockIdx.x, g = threadIdx.x / VT2, ng = blockDim.x / VT2;
    const int b = s.beam, row0 = img * live;
    for (int j = g; j < live; j += ng)
        stats_online128_row(a, row0 + j, threadIdx.x % VT2, GroupBarrier{1 + g}, s_red[g], s_ridx[g], s_val + j * b, s_idx + j * b);
    __syncthreads();
    if (threadIdx.x < 32) select_step<U>(s, img, t, live, b, row0, row0, s_val, s_idx, nullptr, 0, 0.f, penalty_kind, penalty_alpha, done_p);
    if (t == s.T - 1) return;
    __syncthreads();                 // s.src_row of this image is written
    const int n4 = next.H >> 2;
    for (int i = threadIdx.x; i < b * n4; i += blockDim.x) {
        const int j = i / n4, c4 = i - j * n4;
        const long r = (long)img * b + j;
        copy_states4(r, s.src_row[r], c4, 2, next.s0, next.s1);
    }
}

// one warp per real image; its groups step in order, each seeing the words the earlier groups chose at this global step
__global__ void __launch_bounds__(32) diverse_beam_step_kernel(BeamState s, int G, int t, int k, const float* __restrict__ top_val,
                                                               const int* __restrict__ top_idx, float lambda, int rows_total, int penalty_kind,
                                                               float penalty_alpha, double* __restrict__ done_p) {
    const int i = blockIdx.x, lane = threadIdx.x;
    const int b = s.beam, T = s.T;
    __shared__ int sh_pen[MAXB];
    for (int g = 0; g < G && g <= t; ++g) {
        const int lt = t - g;              // the group's local time
        if (lt >= T) continue;             // finished group
        const int n_pen = g * b;
        __syncwarp();                      // the previous group's table writes and shared-memory reads are complete
        if (lane < n_pen) {
            const int pg = lane / b, j = lane - pg * b;
            const int last = min(t - pg, T - 1);       // the last local step of earlier group pg (taken at this t unless it has finished)
            const int* seq_pg = (last & 1) ? s.seq_a : s.seq_b;
            sh_pen[lane] = seq_pg[((long)(i * G + pg) * b + j) * T + lt];
        }
        __syncwarp();
        const int vimg = i * G + g;
        // the group's first step reads the one bos row of the group (its row j = 0), like the B-row first step of beam_step
        select_step(s, vimg, lt, lt == 0 ? 1 : b, k, vimg * b, g * rows_total + vimg * b, top_val + (long)vimg * b * k, top_idx + (long)vimg * b * k,
                    sh_pen, n_pen, lambda, penalty_kind, penalty_alpha, done_p);
    }
}

// one warp per image: stable selection of the `keep` best records by penalised score (CaptionModel.py:207); dynamic shared memory holds one
// `taken` flag per record (beam * T bytes)
__global__ void __launch_bounds__(32) beam_finalize_kernel(BeamState s, int keep, const double* __restrict__ done_p, long long* __restrict__ out_seq,
                                                           int* __restrict__ out_len, float* __restrict__ out_p, float* __restrict__ out_raw,
                                                           int* __restrict__ out_hist) {
    const int img = blockIdx.x, lane = threadIdx.x;
    const int b = s.beam, T = s.T;
    const int cnt = s.done_cnt[img];
    const long base = (long)img * b * T;
    extern __shared__ unsigned char taken[];
    for (int i = lane; i < cnt; i += 32) taken[i] = 0;
    __syncwarp();
    for (int k = 0; k < keep; ++k) {
        double bv = -INFINITY;
        int bi = 0x7fffffff;
        for (int i = lane; i < cnt; i += 32) {
            if (!taken[i]) {
                const double v = done_p[base + i];
                if (v > bv || (v == bv && i < bi)) { bv = v; bi = i; }
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
        }
        const long o = (long)img * keep + k;
        if (bi == 0x7fffffff) {          // fewer records than requested (cannot happen after T steps; keep outputs defined)
            if (lane == 0) { out_len[o] = 0; out_p[o] = -INFINITY; out_raw[o] = -INFINITY; }
            for (int q = lane; q < T; q += 32) { out_seq[o * T + q] = 0; out_hist[o * T + q] = -1; }
            continue;
        }
        if (lane == 0) {
            taken[bi] = 1;
            out_len[o] = s.done_len[base + bi];
            out_p[o] = (float)bv;
            out_raw[o] = s.done_raw[base + bi];
        }
        const int len = s.done_len[base + bi];
        for (int q = lane; q < T; q += 32) {
            out_seq[o * T + q] = (q < len) ? (long long)s.done_seq[(base + bi) * T + q] : 0;
            out_hist[o * T + q] = (q < len) ? s.done_hist[(base + bi) * T + q] : -1;
        }
        __syncwarp();
    }
}

// Decode edits on a per-row candidate list (beam search): the vocabulary kernel delivered the k_in best raw candidates of every row;
// drop / lower the edited ones exactly as the reference edits the log-prob row (CaptionModel.py:154-162) and keep the `beam` best.
// k_in = beam + (number of active edit kinds) guarantees that `beam` unedited candidates remain.  One thread per row.
// Rows with (r % first_beam) / first_group_rows == first_group (diverse beam search: the group starting at this step) are at their first step.
__global__ void beam_edit_kernel(int rows, int k_in, int beam, int t, DecodeEdits ed, const int* __restrict__ prev_tokens,
                                 const float* __restrict__ val_in, const int* __restrict__ idx_in, float* __restrict__ val_out, int* __restrict__ idx_out,
                                 int first_beam, int first_group_rows, int first_group) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    if (first_beam > 0 && (r % first_beam) / first_group_rows == first_group) t = 0;
    float v[MAXB];
    int ix[MAXB];
    const int prev = (t > 0 && prev_tokens != nullptr) ? prev_tokens[r] : -1;
    bool prev_bad = false;
    if (t > 0 && ed.n_bad > 0)
        for (int i = 0; i < ed.n_bad; ++i) prev_bad |= (ed.bad[i] == prev);
    for (int k = 0; k < k_in; ++k) {
        float x = val_in[(long)r * k_in + k];
        const int w = idx_in[(long)r * k_in + k];
        if (ed.constraint && t > 0 && w == prev) x = -INFINITY;
        if (prev_bad && w == 0) x = -INFINITY;
        if (w == ed.unk_col) x -= 1000.0f;
        v[k] = x;
        ix[k] = w;
    }
    // selection sort of the first `beam` (value descending, word index ascending on ties: the order the unedited list came in)
    for (int j = 0; j < beam; ++j) {
        int best = j;
        for (int k = j + 1; k < k_in; ++k)
            if (v[k] > v[best] || (v[k] == v[best] && ix[k] < ix[best])) best = k;
        const float tv = v[j]; v[j] = v[best]; v[best] = tv;
        const int ti = ix[j]; ix[j] = ix[best]; ix[best] = ti;
        val_out[(long)r * beam + j] = v[j];
        idx_out[(long)r * beam + j] = ix[j];
    }
}

__global__ void scale_rows_kernel(float* __restrict__ x, long ld, int rows, int cols, float f, int skip_beam, int skip_group_rows, int skip_group) {
    const long total = (long)rows * cols;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const long r = i / cols, c = i % cols;
        if (skip_beam > 0 && (int)(r % skip_beam) / skip_group_rows == skip_group) continue;
        x[r * ld + c] *= f;
    }
}

__global__ void gather_rows_kernel(const float* __restrict__ slab, long step_stride, long ld_slab, const int* __restrict__ hist, int T, int V1,
                                   float* __restrict__ dst, const float2* __restrict__ stats, long stats_stride, const long long* __restrict__ seqs,
                                   DecodeEdits ed) {
    const long item = blockIdx.x;          // item = k * T + s
    const int sidx = (int)(item % T);
    const int row = hist[item];
    float* d = dst + item * V1;
    if (row < 0) {
        for (int v = threadIdx.x; v < V1; v += blockDim.x) d[v] = 0.f;
        return;
    }
    // the edits the search applied to this row before choosing word `sidx` of this sequence (same stream order: after the row is written)
    auto apply_edits = [&]() {
        if (seqs == nullptr || !ed.any()) return;
        __syncthreads();
        if (threadIdx.x == 0) {
            const int prev = sidx > 0 ? (int)seqs[item - 1] : -1;
            if (ed.unk_col >= 0 && ed.unk_col < V1) d[ed.unk_col] -= 1000.0f;
            if (ed.constraint && prev >= 0 && prev < V1) d[prev] = -INFINITY;
            bool prev_bad = false;
            for (int i = 0; i < ed.n_bad; ++i) prev_bad |= (sidx > 0 && ed.bad[i] == prev);
            if (prev_bad) d[0] = -INFINITY;
        }
    };
    const float* src = slab + (long)sidx * step_stride + (long)row * ld_slab;
    if (stats != nullptr) {
        // raw logits -> log-probs with the row statistics of the search step (second log_softmax from step 1 on)
        const float2 st = stats[(long)sidx * stats_stride + row];
        const float mx = st.x, lsum = st.y;
        const float m2 = (mx - mx) - lsum, l2 = lsum;
        const bool twice = sidx > 0;
        const bool vec4 = ((V1 & 3) == 0) && ((ld_slab & 3) == 0) && ((step_stride & 3) == 0) && ((reinterpret_cast<uintptr_t>(slab) & 15) == 0) &&
                          ((reinterpret_cast<uintptr_t>(dst) & 15) == 0);
        if (vec4) {      // 194 MB of winner rows per decode: 128-bit loads and stores
            const float4* s4 = reinterpret_cast<const float4*>(src);
            float4* d4 = reinterpret_cast<float4*>(d);
            for (int v = threadIdx.x; v < V1 / 4; v += blockDim.x) {
                const float4 x = __ldg(s4 + v);
                float4 o;
                o.x = (x.x - mx) - lsum; o.y = (x.y - mx) - lsum; o.z = (x.z - mx) - lsum; o.w = (x.w - mx) - lsum;
                if (twice) { o.x = (o.x - m2) - l2; o.y = (o.y - m2) - l2; o.z = (o.z - m2) - l2; o.w = (o.w - m2) - l2; }
                d4[v] = o;
            }
        } else {
            for (int v = threadIdx.x; v < V1; v += blockDim.x) {
                const float lp = (src[v] - mx) - lsum;
                d[v] = twice ? (lp - m2) - l2 : lp;
            }
        }
        apply_edits();
        return;
    }
    const bool vec = ((V1 & 3) == 0) && ((ld_slab & 3) == 0) && ((step_stride & 3) == 0) && ((reinterpret_cast<uintptr_t>(slab) & 15) == 0) &&
                     ((reinterpret_cast<uintptr_t>(dst) & 15) == 0);
    if (vec) {
        const float4* s4 = reinterpret_cast<const float4*>(src);
        float4* d4 = reinterpret_cast<float4*>(d);
        for (int v = threadIdx.x; v < V1 / 4; v += blockDim.x) d4[v] = __ldg(s4 + v);
    } else {
        for (int v = threadIdx.x; v < V1; v += blockDim.x) d[v] = src[v];
    }
    apply_edits();
}

}  // namespace

int beam_edit_launch(int rows, int k_in, int beam, int t, const DecodeEdits& ed, const int* prev_tokens, const float* val_in, const int* idx_in,
                     float* val_out, int* idx_out, cudaStream_t stream, int first_beam, int first_group_rows, int first_group) {
    CAPB_REQUIRE(k_in >= beam && k_in <= MAXB, "beam_size + number of active decode edits must be <= 16");
    if (rows <= 0) return 0;
    beam_edit_kernel<<<cdiv(rows, 128), 128, 0, stream>>>(rows, k_in, beam, t, ed, prev_tokens, val_in, idx_in, val_out, idx_out, first_beam,
                                                          first_group_rows, first_group);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int scale_rows_launch(float* x, long ld, int rows, int cols, float factor, cudaStream_t stream, int skip_beam, int skip_group_rows, int skip_group) {
    if (rows <= 0 || cols <= 0) return 0;
    long blocks = ((long)rows * cols + 255) / 256;
    if (blocks > sm_count() * 16) blocks = sm_count() * 16;
    scale_rows_kernel<<<(int)blocks, 256, 0, stream>>>(x, ld, rows, cols, factor, skip_beam, skip_group_rows, skip_group);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int beam_step_launch(const BeamState& s, int t, int live, const float* top_val, const int* top_idx, int penalty_kind, float penalty_alpha,
                     cudaStream_t stream) {
    CAPB_REQUIRE(s.beam >= 1 && s.beam <= MAXB, "beam size 1..16");
    CAPB_REQUIRE(s.beam * s.T <= MAXB * CAPB200_MAX_SEQ_LENGTH, "beam*T record capacity (16 x CAPB200_MAX_SEQ_LENGTH)");
    beam_step_kernel<<<s.B, 32, 0, stream>>>(s, t, live, top_val, top_idx, penalty_kind, penalty_alpha, s.done_p);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

bool beam_search_step_applies(const VocabStepArgs& a, const NextStateGather& next) {
    auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
    auto al8 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7) == 0; };
    auto state_ok = [&](const StateCopy& c) {
        return c.src != nullptr && c.dst.f != nullptr && (c.ld_src & 3) == 0 && (c.dst.ld & 3) == 0 && al16(c.src) && al16(c.dst.f) &&
               ((c.dst.hi == nullptr) == (c.dst.lo == nullptr)) && (c.dst.hi == nullptr || (al8(c.dst.hi) && al8(c.dst.lo)));
    };
    return (a.V1 & 3) == 0 && (a.ld & 3) == 0 && al16(a.logits) && next.H > 0 && (next.H & 3) == 0 && state_ok(next.s0) && state_ok(next.s1);
}

int beam_search_step_launch(const BeamState& s, const VocabStepArgs& a, int t, int live, int penalty_kind, float penalty_alpha,
                            const NextStateGather& next, cudaStream_t stream) {
    CAPB_REQUIRE(s.beam >= 1 && s.beam <= MAXB, "beam size 1..16");
    CAPB_REQUIRE(s.beam * s.T <= MAXB * CAPB200_MAX_SEQ_LENGTH, "beam*T record capacity (16 x CAPB200_MAX_SEQ_LENGTH)");
    CAPB_REQUIRE(a.topk == s.beam && a.stats != nullptr && a.rows == s.B * live && live >= 1 && live <= s.beam, "fused beam step arguments");
    CAPB_REQUIRE(beam_search_step_applies(a, next), "the fused beam step needs 16-byte aligned logit and state rows (V + 1 and H multiples of 4)");
    const int threads = min(live, kStepGroups) * VT2;
    if (s.beam <= 8) beam_search_step_kernel<2><<<s.B, threads, 0, stream>>>(s, a, t, live, penalty_kind, penalty_alpha, s.done_p, next);
    else beam_search_step_kernel<8><<<s.B, threads, 0, stream>>>(s, a, t, live, penalty_kind, penalty_alpha, s.done_p, next);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int diverse_beam_step_launch(const BeamState& s, int G, int t, int k, const float* top_val, const int* top_idx, float lambda, int rows_total,
                             int penalty_kind, float penalty_alpha, cudaStream_t stream) {
    CAPB_REQUIRE(G >= 2 && s.beam >= 1 && G * s.beam <= MAXB, "group_size * beams per group must be in 2..16");
    CAPB_REQUIRE(k >= s.beam && k <= MAXB && s.beam * k <= 256, "candidate list width");
    CAPB_REQUIRE(s.beam * s.T <= MAXB * CAPB200_MAX_SEQ_LENGTH, "beam*T record capacity (16 x CAPB200_MAX_SEQ_LENGTH)");
    CAPB_REQUIRE(lambda >= 0.f, "diversity_lambda must be >= 0 (the candidate lists rely on the penalty only lowering values)");
    diverse_beam_step_kernel<<<s.B / G, 32, 0, stream>>>(s, G, t, k, top_val, top_idx, lambda, rows_total, penalty_kind, penalty_alpha, s.done_p);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int beam_finalize_launch(const BeamState& s, int keep, long long* out_seq, int* out_len, float* out_p, float* out_raw, int* out_hist,
                         cudaStream_t stream) {
    CAPB_REQUIRE(keep >= 1 && keep <= s.beam, "keep must be in 1..beam");
    beam_finalize_kernel<<<s.B, 32, (size_t)s.beam * s.T, stream>>>(s, keep, s.done_p, out_seq, out_len, out_p, out_raw, out_hist);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int gather_logprob_rows_launch(const float* slab, long step_stride, long ld_slab, const int* hist, int nseq, int T, int V1, float* dst,
                               const float2* stats, long stats_stride, cudaStream_t stream, const long long* seqs, const DecodeEdits* ed) {
    if (nseq <= 0) return 0;
    gather_rows_kernel<<<nseq * T, 256, 0, stream>>>(slab, step_stride, ld_slab, hist, T, V1, dst, stats, stats_stride, seqs, ed ? *ed : DecodeEdits());
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace capb200
