// Helpers shared by the engines (UpDown/NewFC in engine.cu, Transformer in tfm_engine.cu, AoA in aoa_engine.cu).
#pragma once
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/capb200.h"
#include "common.cuh"
#include "kernels.cuh"
#include "nvtx.cuh"

// opaque C handle of the CIDEr-D document-frequency table (shared by the UpDown and AoA training steps)
struct capb200_cider_table {
    capb200::CiderTable* t = nullptr;
};

namespace capb200 {

struct Planes {
    __half* hi = nullptr;
    __half* lo = nullptr;
    long ld = 0;
};

// bump allocator over one cudaMalloc'ed block; a dry run (base == nullptr) measures the size
struct Arena {
    char* base = nullptr;
    size_t off = 0;
    template <typename T>
    T* take(size_t n) {
        off = (off + 255) & ~size_t(255);
        T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
        off += n * sizeof(T);
        return p;
    }
};

struct Act {
    ActView v;
    void carve(Arena& a, long rows, long cols, bool planes) {
        v.ld = round_up(cols, 64);          // 128-byte plane rows: every TMA box row is one aligned L2 line
        v.f = a.take<float>(rows * v.ld);
        if (planes) {
            v.hi = a.take<__half>(rows * v.ld);
            v.lo = a.take<__half>(rows * v.ld);
        } else {
            v.hi = v.lo = nullptr;
        }
    }
};

inline DecodeEdits to_edits(const capb200_decode_edits& c) {
    DecodeEdits e;
    e.constraint = c.decoding_constraint;
    e.unk_col = c.unk_col;
    e.n_bad = (c.bad_endings != nullptr && c.n_bad_endings > 0) ? c.n_bad_endings : 0;
    e.bad = c.bad_endings;
    e.trigrams = c.block_trigrams;
    e.trigram_rows = c.trigram_rows;
    return e;
}

inline Planes carve_planes(Arena& a, long rows, long cols) {
    Planes p;
    p.ld = round_up(cols, 64);
    p.hi = a.take<__half>(rows * p.ld);
    p.lo = a.take<__half>(rows * p.ld);
    return p;
}


inline GemmSeg seg_of(const ActView& a, const float* w, long ldw, const Planes& wp, int K) {
    GemmSeg s;
    s.A = a.f; s.lda = a.ld; s.W = w; s.ldw = ldw;
    s.A_hi = a.hi; s.A_lo = a.lo; s.lda_h = a.ld;
    s.W_hi = wp.hi; s.W_lo = wp.lo; s.ldw_h = wp.ld;
    s.K = K;
    return s;
}


// Runs one GEMM in the engine's numeric mode.  `plan` caches the encoded TMA maps of this call site (tensor-core modes);
// `plan_rows` is the row capacity the maps are encoded for, g.M the rows valid in this launch.
inline int run_gemm_mode(int mode, GemmTcPlan** plan, GemmProblem& g, int plan_rows, cudaStream_t st) {
    if (mode == 0) return gemm_simt_launch(g, st);
    if (*plan == nullptr) {
        GemmProblem planned = g;
        planned.M = plan_rows;
        *plan = gemm_tc_plan_create(planned, mode == 1 ? 3 : 1);
        if (*plan == nullptr) return 1;
    }
    return gemm_tc_plan_launch(*plan, &g.epi, g.M, st);
}


// ---------------------------------------------------------------------------------------------------------------------
// Search / sampling state shared by every model family, and the two decode drivers.  A family supplies only its recurrent
// core as a callable:  core(rows, rows_per_image, tokens, src_row, t, logits, ld_logits) -> 0 on success, which must leave the
// step's raw logits [rows, V1] at `logits` (row pitch ld_logits).
// ---------------------------------------------------------------------------------------------------------------------
struct DecodeBuffers {
    int *tokens = nullptr, *src_row = nullptr, *neg1 = nullptr, *unfinished = nullptr, *forced = nullptr;
    float* top_val = nullptr;
    int* top_idx = nullptr;
    float* top_val_e = nullptr;       // [rows, 16] candidate lists after the decode edits (beam search with options)
    int* top_idx_e = nullptr;
    float2* slab_stats = nullptr;     // [T, rows]
    BeamState bs;
    long long* rec_seq = nullptr;     // [B, beam, T] sorted records of the last beam decode
    int *rec_len = nullptr, *rec_hist = nullptr, *out_hist = nullptr, *tmp_len = nullptr;
    float *rec_p = nullptr, *rec_raw = nullptr, *tmp_p = nullptr, *tmp_raw = nullptr;
    float* slab = nullptr;            // separately allocated: [T, rows, V1] raw logits of a beam search
    size_t slab_bytes = 0;
    // diverse beam search: separately allocated, grown on demand: [T + G - 1, rows] row statistics and [B * G] record counts
    float2* dbs_stats = nullptr;
    size_t dbs_stats_bytes = 0;
    int* dbs_done_cnt = nullptr;
    size_t dbs_done_bytes = 0;
    const float2* last_stats = nullptr;   // row statistics of the last beam decode (slab_stats or dbs_stats)
    long slab_step_stride = 0;
    int last_B = 0, last_beam = 0;
    DecodeEdits last_edits;           // edits of the last beam decode (re-applied when a finished beam's rows are materialised later)
    // CUDA graph of the T-step beam loop (every launch of it is static for a given shape / workspace): captured the second time a
    // configuration is seen, replayed afterwards; the launch gaps of ~180 serial kernels are ~5 % of a decode
    cudaGraphExec_t loop_exec = nullptr;
    unsigned long long loop_key[8] = {0, 0, 0, 0, 0, 0, 0, 0}, seen_key[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    long loop_launches = 0;
    bool graph_broken = false;
    // set by beam_decode_driver around a core call whose parent-state gather the previous step's beam_search_step_kernel already did
    bool states_gathered = false;

    void release() {
        if (loop_exec) cudaGraphExecDestroy(loop_exec);
        loop_exec = nullptr;
        cudaFree(slab);
        cudaFree(dbs_stats);
        cudaFree(dbs_done_cnt);
        slab = nullptr; dbs_stats = nullptr; dbs_done_cnt = nullptr;
    }

    void carve(Arena& a, int B, int rows, int beam, int T) {
        tokens = a.take<int>(rows);
        src_row = a.take<int>(rows);
        neg1 = a.take<int>(rows);
        unfinished = a.take<int>(rows);
        forced = a.take<int>(rows);
        top_val = a.take<float>((long)rows * 16);
        top_idx = a.take<int>((long)rows * 16);
        top_val_e = a.take<float>((long)rows * 16);
        top_idx_e = a.take<int>((long)rows * 16);
        slab_stats = a.take<float2>((long)rows * T);
        const long rec = (long)B * beam * T;
        bs.sums = a.take<float>((long)B * beam);
        bs.seq_a = a.take<int>(rec);
        bs.seq_b = a.take<int>(rec);
        bs.hist_a = a.take<int>(rec);
        bs.hist_b = a.take<int>(rec);
        bs.done_cnt = a.take<int>(B);
        bs.done_seq = a.take<int>(rec * T);
        bs.done_hist = a.take<int>(rec * T);
        bs.done_len = a.take<int>(rec);
        bs.done_p = a.take<double>(rec);
        bs.done_raw = a.take<float>(rec);
        bs.tokens = tokens;
        bs.src_row = src_row;
        rec_seq = a.take<long long>(rec);
        rec_hist = a.take<int>(rec);
        out_hist = a.take<int>(rec);
        rec_len = a.take<int>((long)B * beam);
        rec_p = a.take<float>((long)B * beam);
        rec_raw = a.take<float>((long)B * beam);
        tmp_len = a.take<int>((long)B * beam);
        tmp_p = a.take<float>((long)B * beam);
        tmp_raw = a.take<float>((long)B * beam);
    }
};

__global__ void capb_fill_int_kernel(int* p, int n, int v);
__global__ void capb_load_token_column_kernel(const long long* src, long ld, int col, int n, int* dst);
int fill_int_launch(int* p, int n, int v, cudaStream_t st);
int load_token_column_launch(const long long* src, long ld, int col, int n, int* dst, cudaStream_t st);
int store_token_column_launch(const int* src, int n, long long* dst, long ld, int col, cudaStream_t st);

// ancestors of the current rows at step t of a beam search (valid for positions < t): the table beam_step(t-1) wrote
inline const int* beam_ancestors(const BeamState& s, int t) { return ((t - 1) & 1) ? s.hist_a : s.hist_b; }

// AttModel._sample_beam + CaptionModel.beam_search (see engine.cu header for the reference lines)
// Key of everything outside the driver that the captured beam-loop launches depend on (0 disables graph capture)
inline unsigned long long loop_graph_key(const void* ws, const void* wblock, const void* mask, int R, int family) {
    unsigned long long h = 1469598103934665603ull;
    auto mix = [&](unsigned long long v) { h ^= v; h *= 1099511628211ull; };
    mix(reinterpret_cast<uintptr_t>(ws)); mix(reinterpret_cast<uintptr_t>(wblock)); mix(reinterpret_cast<uintptr_t>(mask));
    mix((unsigned long long)R); mix((unsigned long long)family + 17);
    return h | 1ull;
}

// grows a separately allocated device buffer to at least `need` bytes (contents are not kept)
inline int grow_buffer(void** p, size_t* bytes, size_t need, cudaStream_t st) {
    if (need <= *bytes) return 0;
    CAPB_CHECK_CUDA(cudaStreamSynchronize(st));
    if (*p) CAPB_CHECK_CUDA(cudaFree(*p));
    *p = nullptr;
    *bytes = 0;
    const cudaError_t e = cudaMalloc(p, need);
    if (e != cudaSuccess) {
        // not sticky: clear it, or the next launch check of this thread would report it again
        (void)cudaGetLastError();
        *p = nullptr;
        set_error("cannot allocate " + std::to_string(need >> 20) + " MB of device workspace (" + cudaGetErrorString(e) +
                  "); its size grows with batch, length and V + 1: DESIGN.md, 'Vocabularies above 51 199 words'");
        return 1;
    }
    *bytes = need;
    return 0;
}

// Runs a beam loop (`run_loop` enqueues every launch of it on `st`): eagerly the first time `key` is seen, captured into a CUDA graph the
// second time, replayed from the graph afterwards.  `key` covers everything the captured launches depend on.
template <class Loop>
int run_beam_loop(DecodeBuffers& d, const unsigned long long (&key)[8], bool use_graph, long* launches, cudaStream_t st, Loop run_loop) {
    static const bool graphs_off = getenv("CAPB200_NO_GRAPH") != nullptr;
    const bool debug = getenv("CAPB200_GRAPH_DEBUG") != nullptr;
    const bool try_graph = use_graph && !graphs_off && !d.graph_broken;
    if (try_graph && d.loop_exec != nullptr && memcmp(key, d.loop_key, sizeof(key)) == 0) {
        CAPB_CHECK_CUDA(cudaGraphLaunch(d.loop_exec, st));
        *launches += d.loop_launches;
        if (debug) fprintf(stderr, "capb200: beam loop replayed from its CUDA graph\n");
    } else if (try_graph && memcmp(key, d.seen_key, sizeof(key)) == 0) {
        // second decode with this configuration: every lazy initialisation has happened, capture the loop and replay it from now on
        if (d.loop_exec != nullptr) { cudaGraphExecDestroy(d.loop_exec); d.loop_exec = nullptr; }
        const long l0 = *launches;
        cudaGraph_t graph = nullptr;
        bool ok = cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal) == cudaSuccess;
        const int rc = ok ? run_loop() : 1;
        if (ok) ok = cudaStreamEndCapture(st, &graph) == cudaSuccess && graph != nullptr && rc == 0;
        if (ok) ok = cudaGraphInstantiate(&d.loop_exec, graph, 0) == cudaSuccess;
        if (graph != nullptr) cudaGraphDestroy(graph);
        if (!ok) {
            (void)cudaGetLastError();
            d.loop_exec = nullptr;
            d.graph_broken = true;          // fall back to eager launches for good
            *launches = l0;
            if (run_loop()) return 1;
        } else {
            d.loop_launches = *launches - l0;
            memcpy(d.loop_key, key, sizeof(key));
            CAPB_CHECK_CUDA(cudaGraphLaunch(d.loop_exec, st));
            if (debug) fprintf(stderr, "capb200: beam loop captured into a CUDA graph (%ld launches)\n", d.loop_launches);
        }
    } else {
        memcpy(d.seen_key, key, sizeof(key));
        if (run_loop()) return 1;
    }
    return 0;
}

// `next` (optional): the engine's recurrent states, which the core gathers by parent row at the start of every step.  Where it applies
// (no decode edits, temperature 1, 16-byte aligned logit and state rows), each step's vocabulary statistics / top-k, beam step and the
// next step's state gather run as one beam_search_step_kernel per image, and from t = 1 on the core is called with d.states_gathered
// set and skips its own gather: 2T - 1 fewer launches per decode.  `form`: 0 picks that automatically, 1 always runs the separate
// kernels, 2 requires the fused kernel (an error where it does not apply); 1 and 2 are for tests.
template <class CoreFn>
int beam_decode_driver(DecodeBuffers& d, int V1, int T, int B, int beam, int keep, int penalty_kind, float penalty_alpha, long long* seq,
                       float* seq_logprobs, long long* done_seq, int* done_len, float* done_p, float* done_raw, CoreFn core, long* launches,
                       cudaStream_t st, unsigned long long graph_key = 0, const DecodeEdits& ed = DecodeEdits(), float temperature = 1.0f,
                       const NextStateGather* next = nullptr, int form = 0) {
    const int rows = B * beam;
    const bool edits = ed.any();
    const int k_in = beam + ed.kinds();
    CAPB_REQUIRE(!ed.trigrams, "block_trigrams applies to _sample only (AttModel.py:306)");
    CAPB_REQUIRE(k_in <= 16, "beam_size + number of active decode edits (decoding_constraint, remove_bad_endings, UNK suppression) must be <= 16");
    CAPB_REQUIRE(form >= 0 && form <= 2, "beam step form must be 0 (automatic), 1 (separate kernels) or 2 (fused)");
    if (temperature == 0.f) temperature = 1.0f;
    CAPB_REQUIRE(temperature > 0.f, "temperature must be positive");
    if (grow_buffer(reinterpret_cast<void**>(&d.slab), &d.slab_bytes, (size_t)T * rows * V1 * sizeof(float), st)) return 1;
    d.slab_step_stride = (long)rows * V1;
    d.last_B = B;
    d.last_beam = beam;
    BeamState s = d.bs;
    s.B = B; s.beam = beam; s.T = T; s.V1 = V1;
    bool fused = false;
    if (form != 1 && next != nullptr && !edits && temperature == 1.0f) {
        VocabStepArgs probe;            // every step's slab has the alignment of step 0 (V1 % 4 == 0 makes the step stride 16-byte aligned)
        probe.V1 = V1; probe.ld = V1; probe.logits = d.slab;
        fused = beam_search_step_applies(probe, *next);
    }
    CAPB_REQUIRE(form != 2 || fused, "the fused beam step needs the engine's state descriptor, no decode edits, temperature 1 and 16-byte aligned "
                                     "logit and state rows (V + 1 and H multiples of 4)");
    auto run_loop = [&]() -> int {
        CAPB_NVTX("capb200 beam loop (T steps: core, vocab stats, beam step)");
        CAPB_CHECK_CUDA(cudaMemsetAsync(s.sums, 0, sizeof(float) * B * beam, st));
        CAPB_CHECK_CUDA(cudaMemsetAsync(s.done_cnt, 0, sizeof(int) * B, st));
        CAPB_CHECK_CUDA(cudaMemsetAsync(d.tokens, 0, sizeof(int) * rows, st));      // <bos> = 0
        for (int t = 0; t < T; ++t) {
            const int live = (t == 0) ? 1 : beam;
            const int nrows = B * live;
            float* logits = d.slab + (long)t * d.slab_step_stride;
            d.states_gathered = fused && t > 0;
            const int rc = core(nrows, live, d.tokens, t == 0 ? d.neg1 : d.src_row, t, logits, (long)V1);
            d.states_gathered = false;
            if (rc) return 1;
            if (t > 0 && temperature != 1.0f) {      // log_softmax(logprobs / temperature) = log_softmax(logits / temperature)  (CaptionModel.py:204)
                if (scale_rows_launch(logits, V1, nrows, V1, 1.0f / temperature, st)) return 1;
                *launches += 1;
            }
            VocabStepArgs va;
            va.rows = nrows; va.V1 = V1; va.logits = logits; va.ld = V1;
            va.twice = (t > 0) ? 1 : 0;      // init_logprobs went through one log_softmax only (AttModel.py:239, CaptionModel.py:204)
            va.topk = edits ? k_in : beam; va.top_val = d.top_val; va.top_idx = d.top_idx;
            va.stats = d.slab_stats + (long)t * rows;
            if (fused) {
                if (beam_search_step_launch(s, va, t, live, penalty_kind, penalty_alpha, *next, st)) return 1;
                *launches += 1;
                continue;
            }
            if (vocab_step_launch(va, st)) return 1;
            const float* tv = d.top_val;
            const int* ti = d.top_idx;
            if (edits) {      // drop / lower the edited candidates, keep the `beam` best (the edits of CaptionModel.py:154-162)
                if (beam_edit_launch(nrows, k_in, beam, t, ed, d.tokens, d.top_val, d.top_idx, d.top_val_e, d.top_idx_e, st)) return 1;
                tv = d.top_val_e; ti = d.top_idx_e;
                *launches += 1;
            }
            if (beam_step_launch(s, t, live, tv, ti, penalty_kind, penalty_alpha, st)) return 1;
            *launches += 2;
        }
        return 0;
    };
    // graph key: everything the captured launches depend on (caller's key covers workspace / weight / mask pointers and R)
    unsigned long long key[8] = {graph_key, (unsigned long long)B, (unsigned long long)beam, (unsigned long long)T, (unsigned long long)V1,
                                 (unsigned long long)penalty_kind, 0ull, (unsigned long long)reinterpret_cast<uintptr_t>(d.slab)};
    memcpy(&key[6], &penalty_alpha, sizeof(float));
    memcpy(reinterpret_cast<char*>(&key[6]) + 4, &temperature, sizeof(float));
    // decode edits are baked into the captured launches too
    key[5] ^= ((unsigned long long)(ed.constraint & 1) << 8) ^ ((unsigned long long)(unsigned)(ed.unk_col + 1) << 16) ^ ((unsigned long long)ed.n_bad << 48);
    key[5] ^= (unsigned long long)fused << 9;       // and the form of the step
    key[0] ^= (unsigned long long)reinterpret_cast<uintptr_t>(ed.bad) * 0x9E3779B97F4A7C15ull;
    d.last_edits = ed;
    d.last_stats = d.slab_stats;
    if (run_beam_loop(d, key, graph_key != 0, launches, st, run_loop)) return 1;
    // all finished beams of every image, best first
    CAPB_NVTX("capb200 beam finalize + log-prob rows");
    if (beam_finalize_launch(s, beam, d.rec_seq, d.rec_len, d.rec_p, d.rec_raw, d.rec_hist, st)) return 1;
    *launches += 1;
    if (keep == beam) {
        CAPB_CHECK_CUDA(cudaMemcpyAsync(seq, d.rec_seq, sizeof(long long) * B * beam * T, cudaMemcpyDeviceToDevice, st));
        if (seq_logprobs) {
            *launches += 1;
            if (gather_logprob_rows_launch(d.slab, d.slab_step_stride, V1, d.rec_hist, B * beam, T, V1, seq_logprobs, d.slab_stats, rows, st, d.rec_seq, &ed)) return 1;
        }
    } else {
        *launches += 1;
        if (beam_finalize_launch(s, 1, seq, d.tmp_len, d.tmp_p, d.tmp_raw, d.out_hist, st)) return 1;
        if (seq_logprobs) {
            *launches += 1;
            if (gather_logprob_rows_launch(d.slab, d.slab_step_stride, V1, d.out_hist, B, T, V1, seq_logprobs, d.slab_stats, rows, st, seq, &ed)) return 1;
        }
    }
    if (done_seq) CAPB_CHECK_CUDA(cudaMemcpyAsync(done_seq, d.rec_seq, sizeof(long long) * B * beam * T, cudaMemcpyDeviceToDevice, st));
    if (done_len) CAPB_CHECK_CUDA(cudaMemcpyAsync(done_len, d.rec_len, sizeof(int) * B * beam, cudaMemcpyDeviceToDevice, st));
    if (done_p) CAPB_CHECK_CUDA(cudaMemcpyAsync(done_p, d.rec_p, sizeof(float) * B * beam, cudaMemcpyDeviceToDevice, st));
    if (done_raw) CAPB_CHECK_CUDA(cudaMemcpyAsync(done_raw, d.rec_raw, sizeof(float) * B * beam, cudaMemcpyDeviceToDevice, st));
    return 0;
}

// Diverse beam search (AttModel._sample_beam + CaptionModel.beam_search with group_size G > 1): G groups of bdash = beam / G beams, group g
// running its own beam search staggered by g steps, lowered by lambda for every earlier group's beam that holds the same word at the same
// position.  Rows are image-major, row = i*beam + g*bdash + j, and every global step t = 0 .. T+G-2 runs ONE core call over all B*beam rows:
// the rows of groups g >= t are fed <bos> with a fresh state (src_row -1), so a group starting at t == g finds exactly the <bos> step's
// logits in each of its rows, and the rows of groups g < t are fed their chosen word and parent.  Group g's position-p logits are slab step
// p + g: its records' slab rows are g*rows + row, which gather_logprob_rows addresses as slab step p and row statistic p*rows + (g*rows + row).
// The records of (image i, group g) form virtual image i*G + g, so the finalize over B*G virtual images of bdash beams writes done_* in the
// reference's order: each group's records sorted by score, the groups concatenated (CaptionModel.py:207-208).
template <class CoreFn>
int diverse_beam_decode_driver(DecodeBuffers& d, int V1, int T, int B, int beam, int G, float lambda, int keep, int penalty_kind, float penalty_alpha,
                               long long* seq, float* seq_logprobs, long long* done_seq, int* done_len, float* done_p, float* done_raw, CoreFn core,
                               long* launches, cudaStream_t st, unsigned long long graph_key, const DecodeEdits& ed, float temperature) {
    CAPB_REQUIRE(G >= 2 && beam % G == 0, "diverse beam search needs group_size >= 2 dividing beam_size");
    CAPB_REQUIRE(lambda >= 0.f, "diversity_lambda must be >= 0");
    const int bdash = beam / G, rows = B * beam, steps = T + G - 1;
    CAPB_REQUIRE(keep == 1 || keep == bdash, "sample_n must be 1 or beam_size / group_size (AttModel.py:223)");
    const bool edits = ed.any();
    const int k_in = beam + ed.kinds();
    CAPB_REQUIRE(!ed.trigrams, "block_trigrams applies to _sample only (AttModel.py:306)");
    CAPB_REQUIRE(k_in <= 16, "beam_size + number of active decode edits (decoding_constraint, remove_bad_endings, UNK suppression) must be <= 16");
    if (temperature == 0.f) temperature = 1.0f;
    CAPB_REQUIRE(temperature > 0.f, "temperature must be positive");
    if (grow_buffer(reinterpret_cast<void**>(&d.slab), &d.slab_bytes, (size_t)steps * rows * V1 * sizeof(float), st)) return 1;
    if (grow_buffer(reinterpret_cast<void**>(&d.dbs_stats), &d.dbs_stats_bytes, (size_t)steps * rows * sizeof(float2), st)) return 1;
    if (grow_buffer(reinterpret_cast<void**>(&d.dbs_done_cnt), &d.dbs_done_bytes, (size_t)B * G * sizeof(int), st)) return 1;
    d.slab_step_stride = (long)rows * V1;
    d.last_B = B;
    d.last_beam = beam;
    d.last_edits = ed;
    d.last_stats = d.dbs_stats;
    BeamState s = d.bs;              // B*G virtual images of bdash beams over the same [B*beam]-sized tables
    s.B = B * G; s.beam = bdash; s.T = T; s.V1 = V1;
    s.done_cnt = d.dbs_done_cnt;
    auto run_loop = [&]() -> int {
        CAPB_NVTX("capb200 diverse beam loop (T+G-1 steps: core, vocab stats, group steps)");
        CAPB_CHECK_CUDA(cudaMemsetAsync(s.sums, 0, sizeof(float) * rows, st));
        CAPB_CHECK_CUDA(cudaMemsetAsync(s.done_cnt, 0, sizeof(int) * B * G, st));
        CAPB_CHECK_CUDA(cudaMemsetAsync(d.tokens, 0, sizeof(int) * rows, st));          // <bos> = 0
        CAPB_CHECK_CUDA(cudaMemsetAsync(d.src_row, 0xff, sizeof(int) * rows, st));     // -1: fresh zero state until a group starts
        for (int t = 0; t < steps; ++t) {
            float* logits = d.slab + (long)t * d.slab_step_stride;
            if (core(rows, beam, d.tokens, d.src_row, t, logits, (long)V1)) return 1;
            // group t (if any) is at its first step: one log_softmax, no temperature; every other row as at t > 0 of the plain search
            if (t > 0 && temperature != 1.0f) {
                if (scale_rows_launch(logits, V1, rows, V1, 1.0f / temperature, st, beam, bdash, t)) return 1;
                *launches += 1;
            }
            VocabStepArgs va;
            va.rows = rows; va.V1 = V1; va.logits = logits; va.ld = V1;
            va.twice = (t > 0) ? 1 : 0;
            va.first_beam = beam; va.first_group_rows = bdash; va.first_group = t;
            va.topk = edits ? k_in : beam; va.top_val = d.top_val; va.top_idx = d.top_idx;
            va.stats = d.dbs_stats + (long)t * rows;
            if (vocab_step_launch(va, st)) return 1;
            const float* tv = d.top_val;
            const int* ti = d.top_idx;
            if (edits) {
                if (beam_edit_launch(rows, k_in, beam, t, ed, d.tokens, d.top_val, d.top_idx, d.top_val_e, d.top_idx_e, st, beam, bdash, t)) return 1;
                tv = d.top_val_e; ti = d.top_idx_e;
                *launches += 1;
            }
            // the candidate lists hold each row's `beam` best: the penalty lowers at most (G-1)*bdash words, so they contain its bdash best
            if (diverse_beam_step_launch(s, G, t, beam, tv, ti, lambda, rows, penalty_kind, penalty_alpha, st)) return 1;
            *launches += 2;
        }
        return 0;
    };
    unsigned long long key[8] = {graph_key, (unsigned long long)B, (unsigned long long)beam, (unsigned long long)T, (unsigned long long)V1,
                                 (unsigned long long)penalty_kind, 0ull, (unsigned long long)reinterpret_cast<uintptr_t>(d.slab)};
    memcpy(&key[6], &penalty_alpha, sizeof(float));
    memcpy(reinterpret_cast<char*>(&key[6]) + 4, &temperature, sizeof(float));
    key[5] ^= ((unsigned long long)(ed.constraint & 1) << 8) ^ ((unsigned long long)(unsigned)(ed.unk_col + 1) << 16) ^ ((unsigned long long)ed.n_bad << 48);
    key[0] ^= (unsigned long long)reinterpret_cast<uintptr_t>(ed.bad) * 0x9E3779B97F4A7C15ull;
    // a diverse loop never replays a plain one (or one of another group count / lambda) with the same shapes
    unsigned lambda_bits = 0;
    memcpy(&lambda_bits, &lambda, sizeof(float));
    key[3] ^= (1ull << 63) ^ ((unsigned long long)G << 40);
    key[1] ^= (unsigned long long)lambda_bits << 32;
    key[4] ^= (unsigned long long)reinterpret_cast<uintptr_t>(d.dbs_stats) * 0x9E3779B97F4A7C15ull;
    key[2] ^= (unsigned long long)reinterpret_cast<uintptr_t>(d.dbs_done_cnt) << 8;
    if (run_beam_loop(d, key, graph_key != 0, launches, st, run_loop)) return 1;

    CAPB_NVTX("capb200 diverse beam finalize + log-prob rows");
    if (beam_finalize_launch(s, bdash, d.rec_seq, d.rec_len, d.rec_p, d.rec_raw, d.rec_hist, st)) return 1;
    *launches += 1;
    // seq[k] = done_beams[k][0] (group 0's best) for k < B; with sample_n == bdash the rows B .. B*sample_n-1 stay pad with zero log-probs
    // (AttModel.py:241-254 only fills all sample_n rows when sample_n == beam_size)
    CAPB_CHECK_CUDA(cudaMemcpy2DAsync(seq, sizeof(long long) * T, d.rec_seq, sizeof(long long) * beam * T, sizeof(long long) * T, B,
                                      cudaMemcpyDeviceToDevice, st));
    if (keep > 1) CAPB_CHECK_CUDA(cudaMemsetAsync(seq + (long)B * T, 0, sizeof(long long) * (long)B * (keep - 1) * T, st));
    if (seq_logprobs) {
        CAPB_CHECK_CUDA(cudaMemcpy2DAsync(d.out_hist, sizeof(int) * T, d.rec_hist, sizeof(int) * beam * T, sizeof(int) * T, B, cudaMemcpyDeviceToDevice, st));
        *launches += 1;
        if (gather_logprob_rows_launch(d.slab, d.slab_step_stride, V1, d.out_hist, B, T, V1, seq_logprobs, d.dbs_stats, rows, st, seq, &ed)) return 1;
        if (keep > 1) CAPB_CHECK_CUDA(cudaMemsetAsync(seq_logprobs + (long)B * T * V1, 0, sizeof(float) * (long)B * (keep - 1) * T * V1, st));
    }
    if (done_seq) CAPB_CHECK_CUDA(cudaMemcpyAsync(done_seq, d.rec_seq, sizeof(long long) * rows * T, cudaMemcpyDeviceToDevice, st));
    if (done_len) CAPB_CHECK_CUDA(cudaMemcpyAsync(done_len, d.rec_len, sizeof(int) * rows, cudaMemcpyDeviceToDevice, st));
    if (done_p) CAPB_CHECK_CUDA(cudaMemcpyAsync(done_p, d.rec_p, sizeof(float) * rows, cudaMemcpyDeviceToDevice, st));
    if (done_raw) CAPB_CHECK_CUDA(cudaMemcpyAsync(done_raw, d.rec_raw, sizeof(float) * rows, cudaMemcpyDeviceToDevice, st));
    return 0;
}

inline int beam_record_logprobs(DecodeBuffers& d, int V1, int T, int image, int rank, float* dst, cudaStream_t st) {
    CAPB_REQUIRE(d.slab != nullptr && image >= 0 && image < d.last_B && rank >= 0 && rank < d.last_beam, "no such finished beam");
    return gather_logprob_rows_launch(d.slab, d.slab_step_stride, V1, d.rec_hist + ((long)image * d.last_beam + rank) * T, 1, T, V1, dst,
                                      d.last_stats, (long)d.last_B * d.last_beam, st, d.rec_seq + ((long)image * d.last_beam + rank) * T, &d.last_edits);
}

// AttModel._sample (greedy / multinomial / forced replay) and AttModel._forward (teacher forcing); method codes = CAPB200_SAMPLE_*
template <class CoreFn>
int sample_decode_driver(DecodeBuffers& d, int V1, int T, int rows, int method, float temperature, unsigned long long seed, int steps,
                         const long long* tokens_in, long ld_tok, long long* seq, float* seq_logprobs, float* picked, CoreFn core, long* launches,
                         cudaStream_t st, const DecodeEdits& ed = DecodeEdits(), float top = 0.f) {
    const bool teacher = method == 3, forced = method == 2;
    CAPB_NVTX("capb200 sample / teacher-forcing loop");
    CAPB_REQUIRE(ed.unk_col < 0, "UNK suppression is a beam-search option (CaptionModel.py:159-162)");
    if (method == 4) CAPB_REQUIRE(top >= 1.f, "top-k sampling needs k >= 1");
    if (method == 5) CAPB_REQUIRE(top > 0.f && top < 1.f, "nucleus sampling needs 0 < p < 1");
    const long t_out = teacher ? ld_tok : T;
    CAPB_CHECK_CUDA(cudaMemsetAsync(d.tokens, 0, sizeof(int) * rows, st));
    for (int t = 0; t < steps; ++t) {
        if (teacher) { if (load_token_column_launch(tokens_in, ld_tok, t, rows, d.tokens, st)) return 1; *launches += 1; }
        else if (forced) { if (load_token_column_launch(tokens_in, ld_tok, t, rows, d.forced, st)) return 1; *launches += 1; }
        float* logits = seq_logprobs + (long)t * V1;
        if (core(rows, 0, d.tokens, t == 0 ? d.neg1 : nullptr, t, logits, t_out * V1)) return 1;
        VocabStepArgs va;
        va.rows = rows; va.V1 = V1; va.logits = logits; va.ld = t_out * V1;
        va.twice = 0;
        if (!teacher) {
            va.select = (method == 0) ? 1 : (method == 1 ? 2 : (method == 2 ? 3 : method));      // 4 top-k, 5 nucleus
            va.top = top;
            va.edits = ed;
            va.prev_tokens = d.tokens;        // the word fed into this step (read before tokens_out is rewritten at the end of the kernel)
            va.temperature = temperature;
            va.seed = seed;
            va.step = (unsigned long long)t;
            va.forced = d.forced;
            va.unfinished = d.unfinished;
            va.first_step = (t == 0);
            va.tokens_out = d.tokens;
            va.seq_out = seq; va.ld_seq = T; va.t = t;
            va.picked_lp = picked ? picked + t : nullptr;      // picked is [N,T]
            va.ld_picked = T;
        }
        *launches += 1;
        if (vocab_step_launch(va, st)) return 1;
    }
    return 0;
}

// CUDA graph of a whole fused training step (see run_scst_step in train_common.cuh) + the engine-owned staging buffer that gives the graph stable input
// addresses.  CAPB200_SCST_GRAPH=0 keeps the steps eager.
struct StepGraph {
    cudaGraphExec_t exec = nullptr;
    unsigned long long key = 0, seen = 0, cap_seed = 0;
    long launches = 0, replays = 0;
    char* stage = nullptr;
    size_t stage_bytes = 0;
    bool broken = false;
    // The caller's stream is usually torch's legacy default stream, which cannot be captured: the step runs on an engine-owned stream that
    // waits for the caller's stream on entry (enter) and that the caller's stream waits for on exit (leave).
    cudaStream_t stream = nullptr;
    cudaEvent_t ev_in = nullptr, ev_out = nullptr;
    cudaStream_t enter(cudaStream_t caller) {
        if (stream == nullptr) {
            if (cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking) != cudaSuccess || cudaEventCreateWithFlags(&ev_in, cudaEventDisableTiming) != cudaSuccess ||
                cudaEventCreateWithFlags(&ev_out, cudaEventDisableTiming) != cudaSuccess) { (void)cudaGetLastError(); broken = true; return caller; }
        }
        if (cudaEventRecord(ev_in, caller) != cudaSuccess || cudaStreamWaitEvent(stream, ev_in, 0) != cudaSuccess) { (void)cudaGetLastError(); broken = true; return caller; }
        return stream;
    }
    int leave(cudaStream_t caller, cudaStream_t used) {
        if (used == caller) return 0;
        CAPB_CHECK_CUDA(cudaEventRecord(ev_out, used));
        CAPB_CHECK_CUDA(cudaStreamWaitEvent(caller, ev_out, 0));
        return 0;
    }
    static bool enabled() { static const bool v = !(getenv("CAPB200_SCST_GRAPH") != nullptr && atoi(getenv("CAPB200_SCST_GRAPH")) == 0); return v; }
    void reset() { if (exec) cudaGraphExecDestroy(exec); exec = nullptr; key = 0; }
    void destroy() {
        if (getenv("CAPB200_GRAPH_DEBUG") != nullptr && (exec || replays)) fprintf(stderr, "capb200: step graph replayed %ld times\n", replays);
        reset(); if (stage) cudaFree(stage); stage = nullptr; stage_bytes = 0;
        if (ev_in) cudaEventDestroy(ev_in);
        if (ev_out) cudaEventDestroy(ev_out);
        if (stream) cudaStreamDestroy(stream);
        ev_in = ev_out = nullptr; stream = nullptr;
    }
    // copies up to four buffers back to back (256-byte aligned) into the staging buffer in stream order; off[i] = where buffer i landed
    int stage_inputs(int n, const void* const* src, const size_t* bytes, size_t* off, cudaStream_t st) {
        size_t need = 256;
        for (int i = 0; i < n; ++i) { off[i] = need; need += (bytes[i] + 255) & ~size_t(255); }
        if (need > stage_bytes) {
            CAPB_CHECK_CUDA(cudaStreamSynchronize(st));
            reset();
            if (stage) CAPB_CHECK_CUDA(cudaFree(stage));
            stage = nullptr;
            CAPB_CHECK_CUDA(cudaMalloc(&stage, need));
            stage_bytes = need;
        }
        for (int i = 0; i < n; ++i)
            if (src[i] != nullptr && bytes[i]) CAPB_CHECK_CUDA(cudaMemcpyAsync(stage + off[i], src[i], bytes[i], cudaMemcpyDeviceToDevice, st));
        return 0;
    }
    static void mix(unsigned long long& h, const void* p, size_t nbytes) {
        const unsigned char* c = static_cast<const unsigned char*>(p);
        for (size_t i = 0; i < nbytes; ++i) { h ^= c[i]; h *= 1099511628211ull; }
    }
};

// Runs `run()` (which enqueues one whole training step on `st`, reading its inputs from the staging buffer) eagerly the first time `key` is
// seen, captures it into a graph the second time, and replays the graph afterwards with the seed carried by the salt.
template <class Run>
int run_step_graph(StepGraph& sg, unsigned long long key, unsigned long long seed, long* launches, cudaStream_t st, Run run) {
    if (sg.exec != nullptr && sg.key == key) {
        sg.replays++;
        if (dropout_salt_set_all(sg.cap_seed ^ seed, st)) return 1;
        CAPB_CHECK_CUDA(cudaGraphLaunch(sg.exec, st));
        *launches += sg.launches;
        return 0;
    }
    if (dropout_salt_set_all(0ull, st)) return 1;
    if (sg.seen != key) {               // first sighting: eager (it also performs every first-use allocation)
        sg.seen = key;
        return run();
    }
    sg.reset();
    const long l0 = *launches;
    if (cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal) != cudaSuccess) { (void)cudaGetLastError(); sg.broken = true; return run(); }
    const int rc = run();
    cudaGraph_t graph = nullptr;
    const cudaError_t ce = cudaStreamEndCapture(st, &graph);
    if (rc != 0 || ce != cudaSuccess || graph == nullptr) {
        (void)cudaGetLastError();
        if (graph) cudaGraphDestroy(graph);
        sg.broken = true;               // something in the step is not capturable here: stay eager from now on
        *launches = l0;
        return run();
    }
    const cudaError_t ie = cudaGraphInstantiate(&sg.exec, graph, 0);
    cudaGraphDestroy(graph);
    if (ie != cudaSuccess) { (void)cudaGetLastError(); sg.exec = nullptr; sg.broken = true; *launches = l0; return run(); }
    sg.key = key; sg.cap_seed = seed; sg.launches = *launches - l0;
    if (getenv("CAPB200_GRAPH_DEBUG") != nullptr) fprintf(stderr, "capb200: training step captured into a CUDA graph (%ld launches)\n", sg.launches);
    CAPB_CHECK_CUDA(cudaGraphLaunch(sg.exec, st));
    return 0;
}

// Records a caller-owned "gradient group complete" event.  Inside a stream capture (the step is being turned into a graph) the record
// becomes an EXTERNAL event-record node: every replay records the event when the node's dependencies have executed, and a
// cudaStreamWaitEvent issued on another stream after cudaGraphLaunch waits for exactly that (the overlapped all-reduce of grad_sync.py).
inline int record_group_event(cudaEvent_t ev, cudaStream_t st) {
    if (ev == nullptr) return 0;
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    CAPB_CHECK_CUDA(cudaStreamIsCapturing(st, &cs));
    CAPB_CHECK_CUDA(cudaEventRecordWithFlags(ev, st, cs == cudaStreamCaptureStatusActive ? cudaEventRecordExternal : cudaEventRecordDefault));
    return 0;
}

// Side stream of the SCST steps (the eval-mode greedy baseline runs on it while the train-mode sampling pass runs on the caller's stream).
// Lowest priority: both chains are latency-bound and compete for SMs (a persistent GEMM CTA owns its SM's shared memory), and the
// sampling pass is the critical path -- its pending CTAs should be placed first.
inline cudaError_t create_side_stream(cudaStream_t* s) {
    int least = 0, greatest = 0;
    if (cudaDeviceGetStreamPriorityRange(&least, &greatest) == cudaSuccess) return cudaStreamCreateWithPriority(s, cudaStreamNonBlocking, least);
    return cudaStreamCreateWithFlags(s, cudaStreamNonBlocking);
}

// ---------------------------------------------------------------------------------------------------------------------
// The decode workspace of an engine or of the ensemble: one cudaMalloc'ed block holding the family's activations and the DecodeBuffers, and
// the GEMM plans whose tensor maps are encoded on it.
// ---------------------------------------------------------------------------------------------------------------------
struct Workspace {
    char* ws = nullptr;
    size_t ws_bytes = 0;
    int capB = 0, capRows = 0, capR = 0, capBeam = 0;     // extents the block is laid out for (the ensemble's third extent is the caption length)
    DecodeBuffers d;
    std::vector<GemmTcPlan*> plans;                       // per GEMM call site (tensor-core modes)

    void destroy_plans() {
        for (auto& p : plans) { if (p) gemm_tc_plan_destroy(p); p = nullptr; }
    }
    // Grows the block to the largest (B, rows, R, beam) seen so far, laid out by layout(arena, B, rows, R, beam) (a dry run sizes it).  Growing
    // synchronises `st`, drops the plans, zero-fills the new block and sets d.neg1 to all -1.
    template <class Layout>
    int grow(int B, int rows, int R, int beam, cudaStream_t st, Layout layout) {
        if (ws != nullptr && B <= capB && rows <= capRows && R <= capR && beam <= capBeam) return 0;
        const int nB = B > capB ? B : capB, nRows = rows > capRows ? rows : capRows;
        const int nR = R > capR ? R : capR, nBeam = beam > capBeam ? beam : capBeam;
        Arena dry;
        layout(dry, nB, nRows, nR, nBeam);
        const size_t need = dry.off + 256;
        CAPB_CHECK_CUDA(cudaStreamSynchronize(st));
        destroy_plans();
        if (ws) CAPB_CHECK_CUDA(cudaFree(ws));
        ws = nullptr;
        CAPB_CHECK_CUDA(cudaMalloc(&ws, need));
        ws_bytes = need;
        Arena real;
        real.base = ws;
        layout(real, nB, nRows, nR, nBeam);
        capB = nB; capRows = nRows; capR = nR; capBeam = nBeam;
        CAPB_CHECK_CUDA(cudaMemsetAsync(ws, 0, need, st));
        return fill_int_launch(d.neg1, nRows, -1, st);
    }
    void release() {
        destroy_plans();
        cudaFree(ws);
        d.release();
    }
};

// What a family's core reads besides its rows: the batch, the region count it runs with, their mask, and under teacher forcing the token
// matrix (the Transformer masks its pad keys with it).
struct DecodeCtx {
    int B = 0, R = 0;
    const float* mask = nullptr;
    const long long* labels = nullptr;
    long ld_labels = 0;
};

// ---------------------------------------------------------------------------------------------------------------------
// What every engine owns -- capb200_engine (UpDown, Att2in2, NewFC: engine.cu), capb200_aoa_engine (aoa_engine.cu) and capb200_tfm_engine
// (tfm_engine.cu) -- and the three hooks every eval-mode decode is built from: workspace sizing for `rows` rows, the prologue
// (_prepare_feature) for B images, and one application of the recurrent core.  The single-model decodes below and the test-time ensemble
// (ensemble.cu) run the same three.
// ---------------------------------------------------------------------------------------------------------------------
struct EngineBase : Workspace {
    int V1 = 0, T = 0, mode = 0;
    bool tc = false, bound = false;
    long launches = 0;
    const char* bind_name = "";      // the family's bind entry point, named when it has not been called
    int family = -1;                 // CAPB200_FAMILY_* as an ensemble member declares it (-1: the Transformer, which is never one)
    int graph_family = 0;            // the family's term of loop_graph_key
    bool reads_fc = false;           // the decode reads the fc features (UpDown, NewFC)
    bool reads_att = true;           // ... and the regions; a family without them runs with R = 1 (NewFC)
    int max_teacher_steps = 1 << 30; // teacher-forced positions the core holds (the Transformer's cache: T + 1)

    char* wblock = nullptr;          // bind-time buffers
    size_t wblock_bytes = 0;
    char* tape = nullptr;            // training tape, grown on demand
    size_t tape_bytes = 0;
    Tf32Context* tf32 = nullptr;     // tensor maps + transposed operands of the training GEMMs (tensor-core modes)
    static constexpr int kMaxGradGroups = 10;
    cudaEvent_t grad_events[kMaxGradGroups] = {};   // caller-owned: recorded when a gradient group is complete (*_set_grad_events)
    int grad_groups = 2;             // the family's gradient groups: 2, AoANet 10
    cudaStream_t side = nullptr;     // the SCST step's concurrent greedy baseline runs here
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    StepGraph sg;                    // CUDA graph of the whole SCST step

    // AttModel's output head with logit_layers = k > 1 (AttModel.py:87-92): k - 1 hidden Linear(H, H) + ReLU layers between the core's
    // output and the vocabulary projection, outside the recurrence.  Their Dropout(0.5) is a train-mode op, so no decode applies it.
    int logit_layers = 1;
    int head_H = 0;
    int head_site0 = 0;                          // GEMM call site of hidden layer 0; layer i runs at head_site0 + i
    std::vector<const float*> head_w, head_b;    // [k - 1] the caller's fp32 weights [H, H] and biases [H]
    std::vector<Planes> head_planes;             // their split fp16 planes (tensor-core modes), in head_block
    char* head_block = nullptr;
    bool head_bound = false;
    Act head_act[2];                             // the hidden activations [rows, H] of the decode workspace, layer i in head_act[i & 1]
    // training: the gradient buffers of the hidden layers (group 0, with the vocabulary Linear), the dropout rate of the next training calls
    // (AttModel's Dropout(0.5) in train mode, 0 in eval mode), and the tape of the k - 1 post-dropout activations [N, T, H] plus two
    // gradient scratch slabs of the same size, grown on demand
    std::vector<float*> head_gw, head_gb;
    bool head_grads_bound = false;
    float head_drop = 0.5f;
    float* head_tape = nullptr;
    size_t head_tape_bytes = 0;

    virtual ~EngineBase() {
        release();
        cudaFree(head_block);
        cudaFree(head_tape);
        cudaFree(wblock);
        cudaFree(tape);
        sg.destroy();
        tf32_context_destroy(tf32);
        if (ev_fork) cudaEventDestroy(ev_fork);
        if (ev_join) cudaEventDestroy(ev_join);
        if (side) cudaStreamDestroy(side);
    }
    // rows_per_image: the rows of one image in the first core call (NewFC feeds each row its image's embedding there)
    virtual int decode_workspace(int B, int rows, int R, int beam, int rows_per_image, cudaStream_t st) = 0;
    virtual int decode_prepare(const float* fc, const float* att, const DecodeCtx& c, cudaStream_t st) = 0;
    // src_row: parent row per row -- d.neg1 a fresh zero state, null the row itself (sampling from t = 1 on)
    virtual int decode_core(int rows, int rpi, const int* tokens, const int* src_row, int t, float* logits, long ld, const DecodeCtx& c,
                            cudaStream_t st) = 0;
    // the states the fused beam step may gather for the next core call (UpDown), after decode_workspace
    virtual bool next_state(NextStateGather*) { return false; }
    // whether the beam loop may be captured into a graph (not while the LSTM engine times its GEMMs: per-launch events are not captured)
    virtual bool loop_graph_ok() const { return true; }

    // one GEMM in the engine's numeric mode at call site `site`
    int gemm(int site, GemmProblem& g, int plan_rows, cudaStream_t st) {
        launches++;
        return run_gemm_mode(mode, &plans[site], g, plan_rows, st);
    }
    // the split fp16 planes of a weight [rows, cols]
    int pack(const float* w, long ldw, int rows, int cols, const Planes& p, cudaStream_t st) {
        launches++;
        return split_planes_launch(w, ldw, rows, cols, p.hi, p.lo, p.ld, st);
    }
    // LSTM weight blocks [4H, cols] are stored gate-interleaved (row 4*j+g) so the GEMM epilogue can apply the cell directly
    int pack_gates(const float* w, long ldw, int H, int cols, const Planes& p, cudaStream_t st) {
        launches++;
        return split_planes_interleave_launch(w, ldw, H, cols, p.hi, p.lo, p.ld, st);
    }
    // the weight block, allocated and zero-filled on the first bind and laid out by layout(arena) (a dry run sizes it)
    template <class Layout>
    int alloc_wblock(cudaStream_t st, Layout layout) {
        if (wblock != nullptr) return 0;
        Arena dry;
        layout(dry);
        wblock_bytes = dry.off + 256;
        CAPB_CHECK_CUDA(cudaMalloc(&wblock, wblock_bytes));
        CAPB_CHECK_CUDA(cudaMemsetAsync(wblock, 0, wblock_bytes, st));
        Arena real;
        real.base = wblock;
        layout(real);
        return 0;
    }
    // The end of a bind.  The first one waits for the conversions and refuses weights outside the fp16 range of the split planes.  Re-bindings
    // (a training loop changes the weights every step) must not stall the host: the range flag is host-mapped and every later entry point
    // checks it (check_ready), so an overflow introduced by an optimizer step is reported by the next call instead.
    int finish_bind(cudaStream_t st) {
        if (tc && !bound) {
            CAPB_CHECK_CUDA(cudaStreamSynchronize(st));
            CAPB_CHECK_RANGE();
        }
        bound = true;
        return 0;
    }

    // ---- the logit head (logit_layers > 1) ----
    // The depth is fixed before the first decode: the workspace and the GEMM call sites are laid out for it.
    int set_logit_layers(int k, int H) {
        CAPB_REQUIRE(k >= 1, "logit_layers must be >= 1");
        if (k == logit_layers) return 0;
        CAPB_REQUIRE(logit_layers == 1 && ws == nullptr, "logit_layers is set once, before the first decode");
        logit_layers = k;
        head_H = H;
        head_site0 = (int)plans.size();
        plans.resize(plans.size() + k - 1, nullptr);
        head_w.assign(k - 1, nullptr);
        head_b.assign(k - 1, nullptr);
        head_planes.assign(k - 1, Planes());
        head_gw.assign(k - 1, nullptr);
        head_gb.assign(k - 1, nullptr);
        return 0;
    }
    // The gradient buffers gw[i] [H, H] and gb[i] [H] of hidden layer i, OVERWRITTEN by every training call that follows.
    int bind_logit_head_grads(float* const* gw, float* const* gb) {
        const int n = logit_layers - 1;
        CAPB_REQUIRE(n >= 1, "the engine has no hidden head layers: set logit_layers > 1 first");
        CAPB_REQUIRE(gw != nullptr && gb != nullptr, "null argument");
        for (int i = 0; i < n; ++i) CAPB_REQUIRE(gw[i] != nullptr && gb[i] != nullptr, "missing logit head gradient buffers");
        for (int i = 0; i < n; ++i) { head_gw[i] = gw[i]; head_gb[i] = gb[i]; }
        head_grads_bound = true;
        return 0;
    }
    int set_logit_dropout(float p) {
        CAPB_REQUIRE(p >= 0.f && p < 1.f, "the logit head's dropout rate must be in [0, 1)");
        head_drop = p;
        return 0;
    }
    // (Re)binds the hidden layers' weights w[i] [H, H] and biases b[i] [H], i < k - 1; tensor-core modes repack their planes.
    int bind_logit_head(const float* const* w, const float* const* b, cudaStream_t st) {
        const int n = logit_layers - 1, H = head_H;
        CAPB_REQUIRE(n >= 1, "the engine has no hidden head layers: set logit_layers > 1 first");
        CAPB_REQUIRE(w != nullptr && b != nullptr, "null argument");
        for (int i = 0; i < n; ++i) CAPB_REQUIRE(w[i] != nullptr && b[i] != nullptr, "missing logit head weights");
        if (tc && head_block == nullptr) {
            Arena dry;
            for (int i = 0; i < n; ++i) carve_planes(dry, H, H);
            CAPB_CHECK_CUDA(cudaMalloc(&head_block, dry.off + 256));
            Arena real;
            real.base = head_block;
            for (int i = 0; i < n; ++i) head_planes[i] = carve_planes(real, H, H);
        }
        for (int i = 0; i < n; ++i) {
            head_w[i] = w[i];
            head_b[i] = b[i];
            if (tc && pack(w[i], H, H, H, head_planes[i], st)) return 1;
        }
        head_bound = true;
        return 0;
    }
    // the hidden activations in a decode workspace of `rows` rows
    void carve_head(Arena& a, long rows) {
        if (logit_layers > 1)
            for (Act& h : head_act) h.carve(a, rows, head_H, tc);
    }
    // The hidden layers on `rows` rows of the core's output `x`; *out = what the vocabulary GEMM reads (x itself when k = 1).  Each layer is
    // one GEMM whose epilogue adds the bias, applies the ReLU and stores the fp32 row with its split planes.
    int run_logit_head(const ActView& x, int rows, ActView* out, cudaStream_t st) {
        ActView in = x;
        for (int i = 0; i + 1 < logit_layers; ++i) {
            const ActView& y = head_act[i & 1].v;
            GemmProblem g;
            g.M = rows; g.N = head_H; g.nseg = 1;
            g.seg[0] = seg_of(in, head_w[i], head_H, head_planes[i], head_H);
            g.epi.bias = head_b[i]; g.epi.relu = 1;
            g.epi.C = y.f; g.epi.ldc = y.ld; g.epi.C_hi = y.hi; g.epi.C_lo = y.lo; g.epi.ldcs = y.ld;
            if (gemm(head_site0 + i, g, capRows, st)) return 1;
            in = y;
        }
        *out = in;
        return 0;
    }
};

// The checks every engine's create makes after its family's own, and the engine with the shared fields set (`sites` GEMM call sites); null
// after an error.
template <class Engine>
Engine* create_engine(int vocab_size, int seq_length, int numeric_mode, int sites) {
    if (numeric_mode < 0 || numeric_mode > 2) { set_error("unknown numeric mode"); return nullptr; }
    if (seq_length < 1 || seq_length > CAPB200_MAX_SEQ_LENGTH) { set_error("seq_length must be in 1..256 (CAPB200_MAX_SEQ_LENGTH)"); return nullptr; }
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { set_error("no CUDA device: the capb200 engine has no CPU fallback"); return nullptr; }
    Engine* e = new Engine();
    e->V1 = vocab_size + 1;
    e->T = seq_length;
    e->mode = numeric_mode;
    e->tc = numeric_mode != CAPB200_MODE_SIMT_FP32;
    e->plans.assign(sites, nullptr);
    return e;
}

// The per-token gate table of an LSTM whose word enters through the W_ih columns `w_x` (planes p_x): relu(embed)[V+1, E] * w_x^T into
// xgate [V+1, ld_xgate].  One GEMM per bind; it replaces a K = E segment in every decode step (engine.cu).
int build_gate_table(EngineBase& e, const float* embed, int E, int H, const float* w_x, long ld_w, const Planes& p_x, float* xgate, long ld_xgate,
                     cudaStream_t st);
int add_vec_launch(const float* a, const float* b, float* o, int n, cudaStream_t st);
int interleave_gates_launch(const float* src, float* dst, int H, cudaStream_t st);      // dst[4*j+g] = src[g*H + j]

// The engine behind an ensemble member's handle (engine.cu, aoa_engine.cu)
EngineBase* engine_base(capb200_engine* e);
EngineBase* engine_base(capb200_aoa_engine* e);

inline int check_ready(const EngineBase* e) {
    CAPB_REQUIRE(e != nullptr, "null engine");
    CAPB_REQUIRE(e->bound, std::string(e->bind_name) + " has not been called");
    CAPB_REQUIRE(e->logit_layers == 1 || e->head_bound, "the logit head (logit_layers > 1) has not been bound");
    CAPB_CHECK_RANGE();
    return 0;
}

// The training steps and the autograd entry points write the head's gradients too: they need its buffers.
inline int check_train_ready(const EngineBase* e) {
    if (check_ready(e)) return 1;
    CAPB_REQUIRE(e->logit_layers == 1 || e->head_grads_bound, "the logit head's gradient buffers (logit_layers > 1) have not been bound");
    return 0;
}

inline int set_grad_events(EngineBase* e, void* const* events, int n) {
    CAPB_REQUIRE(e != nullptr, "null engine");
    CAPB_REQUIRE(n >= 0 && n <= e->grad_groups, "the engine has " + std::to_string(e->grad_groups) + " gradient groups");
    for (int i = 0; i < e->grad_groups; ++i) e->grad_events[i] = (events != nullptr && i < n) ? static_cast<cudaEvent_t>(events[i]) : nullptr;
    return 0;
}

// ---- the argument checks of the decode entry points (the engines' and the ensemble's) -------------------------------------------------------
// beam_size and sample_n of a beam search; with group_size > 1 (`diverse`) the driver checks sample_n against beam_size / group_size
inline int check_beam_opts(const capb200_beam_opts* o, int V1, const long long* seq, bool diverse = false) {
    CAPB_REQUIRE(o != nullptr && seq != nullptr, "null argument");
    const int beam = o->beam_size;
    if (diverse) {
        CAPB_REQUIRE(beam >= 2 && beam <= 16 && beam <= V1, "beam_size must be in 2..16 and <= V+1");
        return 0;
    }
    CAPB_REQUIRE(beam >= 1 && beam <= 16 && beam <= V1, "beam_size must be in 1..16 and <= V+1");
    CAPB_REQUIRE(o->sample_n == 1 || o->sample_n == beam, "sample_n must be 1 or beam_size (AttModel.py:223)");
    return 0;
}

// sampling / teacher forcing; *steps = the positions to run (T, or opts->steps under teacher forcing)
inline int check_sample_opts(const capb200_sample_opts* o, int B, int T, int max_teacher_steps, const long long* tokens_in, long ld_tok,
                             const long long* seq, const float* seq_logprobs, int* steps) {
    CAPB_REQUIRE(o != nullptr && seq_logprobs != nullptr, "null argument");
    const int method = o->method;
    CAPB_REQUIRE(o->sample_n >= 1 && B >= 1, "empty batch");
    CAPB_REQUIRE(method >= 0 && method <= 5, "unknown sampling method");
    const bool teacher = method == CAPB200_SAMPLE_TEACHER;
    if (method == CAPB200_SAMPLE_FORCED || teacher) CAPB_REQUIRE(tokens_in != nullptr && ld_tok >= 1, "token matrix required");
    if (!teacher) CAPB_REQUIRE(seq != nullptr, "seq output required");
    if (method == CAPB200_SAMPLE_MULTINOMIAL || method >= CAPB200_SAMPLE_TOPK) CAPB_REQUIRE(o->temperature > 0.f, "temperature must be positive");
    *steps = teacher ? o->steps : T;
    CAPB_REQUIRE(*steps >= 0 && *steps <= (teacher ? ld_tok : T) && *steps <= max_teacher_steps, "steps out of range");
    return 0;
}

// the features an engine's decode reads
inline int check_decode_feats(const EngineBase& e, const float* fc, const float* att, int B, int* R) {
    CAPB_REQUIRE(B >= 1, "empty batch");
    CAPB_REQUIRE(fc != nullptr || !e.reads_fc, "fc features required");
    if (!e.reads_att) *R = 1;
    else CAPB_REQUIRE(att != nullptr && *R >= 1, "attention features required");
    return 0;
}

// ---- the decode entry points of every engine: the checks, the family's three hooks, the driver ----------------------------------------------
inline unsigned long long engine_loop_key(EngineBase* e, const float* mask, int R) {
    return e->loop_graph_ok() ? loop_graph_key(e->ws, e->wblock, mask, R, e->graph_family) : 0ull;
}

inline int decode_beam(EngineBase* e, const float* fc, const float* att, const float* mask, int B, int R, const capb200_beam_opts* opts, long long* seq,
                       float* seq_logprobs, long long* done_seq, int* done_len, float* done_p, float* done_raw, cudaStream_t st, int form = 0) {
    if (check_ready(e) || check_beam_opts(opts, e->V1, seq) || check_decode_feats(*e, fc, att, B, &R)) return 1;
    const int beam = opts->beam_size;
    const DecodeCtx c{B, R, mask};
    if (e->decode_workspace(B, B * beam, R, beam, 1, st) || e->decode_prepare(fc, att, c, st)) return 1;
    auto core = [&](int rows, int rpi, const int* tokens, const int* src_row, int t, float* logits, long ld) {
        return e->decode_core(rows, rpi, tokens, src_row, t, logits, ld, c, st);
    };
    NextStateGather next;
    const bool gather = e->next_state(&next);
    return beam_decode_driver(e->d, e->V1, e->T, B, beam, opts->sample_n, opts->penalty_kind, opts->penalty_alpha, seq, seq_logprobs, done_seq, done_len,
                              done_p, done_raw, core, &e->launches, st, engine_loop_key(e, mask, R), to_edits(opts->edits), opts->temperature,
                              gather ? &next : nullptr, form);
}

inline int decode_beam_diverse(EngineBase* e, const float* fc, const float* att, const float* mask, int B, int R, const capb200_diverse_opts* opts,
                               long long* seq, float* seq_logprobs, long long* done_seq, int* done_len, float* done_p, float* done_raw, cudaStream_t st) {
    if (check_ready(e)) return 1;
    CAPB_REQUIRE(opts != nullptr, "null argument");
    // NewFC picks its fresh-state pass (the image embedding step) per core call, not per row, so its groups cannot start at different steps
    CAPB_REQUIRE(e->reads_att, "diverse beam search needs a family that attends over regions (NewFC's fresh-state pass is chosen per call, not per row)");
    if (opts->group_size == 1) return decode_beam(e, fc, att, mask, B, R, &opts->base, seq, seq_logprobs, done_seq, done_len, done_p, done_raw, st);
    if (check_beam_opts(&opts->base, e->V1, seq, true) || check_decode_feats(*e, fc, att, B, &R)) return 1;
    const int beam = opts->base.beam_size;
    const DecodeCtx c{B, R, mask};
    if (e->decode_workspace(B, B * beam, R, beam, 1, st) || e->decode_prepare(fc, att, c, st)) return 1;
    auto core = [&](int rows, int rpi, const int* tokens, const int* src_row, int t, float* logits, long ld) {
        return e->decode_core(rows, rpi, tokens, src_row, t, logits, ld, c, st);
    };
    return diverse_beam_decode_driver(e->d, e->V1, e->T, B, beam, opts->group_size, opts->diversity_lambda, opts->base.sample_n, opts->base.penalty_kind,
                                      opts->base.penalty_alpha, seq, seq_logprobs, done_seq, done_len, done_p, done_raw, core, &e->launches, st,
                                      engine_loop_key(e, mask, R), to_edits(opts->base.edits), opts->base.temperature);
}

inline int decode_record_logprobs(EngineBase* e, int image, int rank, float* dst, cudaStream_t st) {
    if (check_ready(e)) return 1;
    return beam_record_logprobs(e->d, e->V1, e->T, image, rank, dst, st);
}

inline int decode_sample(EngineBase* e, const float* fc, const float* att, const float* mask, int B, int R, const capb200_sample_opts* opts,
                         const long long* tokens_in, long ld_tok, long long* seq, float* seq_logprobs, float* picked, cudaStream_t st) {
    int steps = 0;
    if (check_ready(e) || check_sample_opts(opts, B, e->T, e->max_teacher_steps, tokens_in, ld_tok, seq, seq_logprobs, &steps) ||
        check_decode_feats(*e, fc, att, B, &R)) return 1;
    const int n = opts->sample_n, rows = B * n;
    const DecodeCtx c{B, R, mask, opts->method == CAPB200_SAMPLE_TEACHER ? tokens_in : nullptr, ld_tok};
    if (e->decode_workspace(B, rows, R, 1, n, st) || e->decode_prepare(fc, att, c, st)) return 1;
    auto core = [&](int nrows, int /*live*/, const int* tokens, const int* src_row, int t, float* logits, long ld) {
        return e->decode_core(nrows, n, tokens, src_row, t, logits, ld, c, st);
    };
    return sample_decode_driver(e->d, e->V1, e->T, rows, opts->method, opts->temperature, opts->seed, steps, tokens_in, ld_tok, seq, seq_logprobs,
                                picked, core, &e->launches, st, to_edits(opts->edits), opts->top);
}

// Training-step GEMMs on the raw fp32 PyTorch weights (always current, no repack after optimizer steps).  With a Tf32Context (tensor-core
// engines) every call runs on the wgmma tf32 3-pass kernel of gemm_tf32.cu; operands that are not K-major in HBM (W for the input
// gradients, dY / X for the weight gradients) go through cached transposes.  Without a context (simt_fp32 engines), or when an operand is
// not TMA-compatible (rows not 16-byte aligned: tiny test shapes), the split-K kernels of gemm_generic.cu run.
struct Skinny {
    float* scratch; size_t cap; int mode; cudaStream_t st;
    Tf32Context* ctx = nullptr;
    bool tc() const { return ctx != nullptr && mode != 0; }
    // y = x * W^T (+ b)          (nn.Linear forward; W stored [N, K])
    int lin(const float* x, long ldx, const float* w, long ldw, const float* b, float* y, long ldy, int M, int N, int K, int accumulate) const {
        if (tc() && gemm_tf32_supported(1, &x, &ldx, &w, &ldw, &K))
            return gemm_tf32_launch(ctx, M, N, 1, &x, &ldx, &w, &ldw, &K, y, ldy, b, nullptr, 0, 1, accumulate, st);
        const int tb = 1;
        return gemm_skinny_launch(M, N, 1, &x, &ldx, &w, &ldw, &K, &tb, y, ldy, b, nullptr, 0, 1, accumulate, scratch, cap, mode, st);
    }
    // dx = dy * W                (nn.Linear input gradient; W stored [K, N] = [out, in])
    int dgrad(int M, int N, int K, const float* dy, long lddy, const float* w, long ldw, float* dx, long lddx, int accumulate) const {
        if (tc() && (reinterpret_cast<uintptr_t>(dy) & 15) == 0 && (lddy & 3) == 0) {
            long ldt = 0;
            const float* wt = tf32_transposed(ctx, w, ldw, K, N, true, &ldt, st);          // W^T [N, K]: rebuilt once per training step
            if (wt == nullptr) return 1;
            return gemm_tf32_launch(ctx, M, N, 1, &dy, &lddy, &wt, &ldt, &K, dx, lddx, nullptr, nullptr, 0, 1, accumulate, st);
        }
        const int tb = 0;
        return gemm_skinny_launch(M, N, 1, &dy, &lddy, &w, &ldw, &K, &tb, dx, lddx, nullptr, nullptr, 0, 1, accumulate, scratch, cap, mode, st);
    }
    // the K-segmented gate GEMM of the decode path, on fp32 weights
    int gates(const GemmProblem& g) const {
        const float* A[3]; const float* B[3]; long lda[3], ldb[3]; int K[3], tb[3];
        for (int i = 0; i < g.nseg; ++i) { A[i] = g.seg[i].A; lda[i] = g.seg[i].lda; B[i] = g.seg[i].W; ldb[i] = g.seg[i].ldw; K[i] = g.seg[i].K; tb[i] = 1; }
        if (tc() && gemm_tf32_supported(g.nseg, A, lda, B, ldb, K))
            return gemm_tf32_launch(ctx, g.M, g.N, g.nseg, A, lda, B, ldb, K, g.epi.C, g.epi.ldc, g.epi.bias, g.epi.row_bias, g.epi.ld_row_bias,
                                    g.epi.rows_per_group, 0, st);
        return gemm_skinny_launch(g.M, g.N, g.nseg, A, lda, B, ldb, K, tb, g.epi.C, g.epi.ldc, g.epi.bias, g.epi.row_bias, g.epi.ld_row_bias,
                                  g.epi.rows_per_group, 0, scratch, cap, mode, st);
    }
    // dW[out, in] (+)= dY[rows, out]^T * X[rows, in]      (weight gradient, batched over time: rows = T * N)
    int wgrad(int out_f, int in_f, int rows, const float* dY, long ld_dy, const float* X, long ld_x, float* G, long ld_g, int accumulate) const {
        if (tc() && rows >= 64) {
            long ld_a = 0, ld_b = 0;
            const float* dyt = tf32_transposed(ctx, dY, ld_dy, rows, out_f, false, &ld_a, st);     // [out, rows]
            const float* xt = dyt ? tf32_transposed(ctx, X, ld_x, rows, in_f, false, &ld_b, st) : nullptr;     // [in, rows]
            if (xt == nullptr) return 1;
            return gemm_tf32_launch(ctx, out_f, in_f, 1, &dyt, &ld_a, &xt, &ld_b, &rows, G, ld_g, nullptr, nullptr, 0, 1, accumulate, st);
        }
        return gemm_wgrad_launch(out_f, in_f, rows, dY, ld_dy, X, ld_x, G, ld_g, accumulate, mode, st);
    }
};


}  // namespace capb200
