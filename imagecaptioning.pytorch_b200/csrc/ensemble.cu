// Test-time ensemble: AttEnsemble (captioning/models/AttEnsemble.py) on the engine.  C ABI capb200_ensemble_* in include/capb200.h.
//
// Every step runs each member's own recurrent core (the decode pieces of engine.cu / aoa_engine.cu) on the same rows, input words and parent
// rows into an ensemble-owned [K, rows, V+1] block of raw logits; one mixing pass then writes
//     log( sum_k softmax(z_k) * w_k / sum_k w_k )                              AttEnsemble.get_logprobs_state :50-58
// where a single model's core leaves its logits.  The beam and sampling drivers of engine_common.cuh run on that row unchanged: their
// log_softmax passes and the temperature scaling act on it as on a single model's logits (a log_softmax of a normalised row returns it, up
// to rounding).  Each member keeps its own workspace and runs its own prologue (_prepare_feature) once per call.
#include <cmath>

#include "../../include/capb200.h"
#include "common.cuh"
#include "engine_common.cuh"
#include "kernels.cuh"

using namespace capb200;

struct capb200_ensemble : Workspace {      // the DecodeBuffers of the ensemble's searches
    float* mix = nullptr;        // [K, rows, V+1] member logits of one step
    size_t mix_bytes = 0;
    int V1 = 0, T = 0;           // of the last decode (capb200_ensemble_beam_record_logprobs)
    long launches = 0;
};

namespace capb200 {

constexpr int kMixThreads = 256;

struct MixWeights {
    float w[CAPB200_ENSEMBLE_MAX_MEMBERS];
    float sum;
    int K;
};

// merges the partial row statistics (m2, s2) into (m, s): running max and sum of exp(x - max)
__device__ __forceinline__ void lse_merge(float& m, float& s, float m2, float s2) {
    if (m2 == -INFINITY) return;
    if (m == -INFINITY) { m = m2; s = s2; return; }
    if (m2 > m) { s = s * expf(m - m2) + s2; m = m2; }
    else s += s2 * expf(m2 - m);
}

// One CTA per row: a max / sum-of-exp pass over each member's logits, then one pass that writes the mixture in the reference's fp32 order
// (softmax(z_k) * w_k, / sum w, summed over k in member order, log).  z: [K][rows][V1] with member pitch member_stride.
__global__ void __launch_bounds__(kMixThreads) capb_ensemble_mix_kernel(const float* __restrict__ z, long member_stride, int V1, MixWeights mw,
                                                                        float* __restrict__ out, long ld_out) {
    __shared__ float red_m[kMixThreads / 32], red_s[kMixThreads / 32];
    __shared__ float row_m[CAPB200_ENSEMBLE_MAX_MEMBERS], row_s[CAPB200_ENSEMBLE_MAX_MEMBERS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const float* zr = z + (long)blockIdx.x * V1;
    for (int k = 0; k < mw.K; ++k) {
        const float* zk = zr + k * member_stride;
        float m = -INFINITY, s = 0.f;
        for (int v = threadIdx.x; v < V1; v += kMixThreads) lse_merge(m, s, zk[v], 1.f);
        for (int o = 16; o > 0; o >>= 1) lse_merge(m, s, __shfl_xor_sync(0xffffffffu, m, o), __shfl_xor_sync(0xffffffffu, s, o));
        if (lane == 0) { red_m[warp] = m; red_s[warp] = s; }
        __syncthreads();
        if (warp == 0) {
            m = lane < kMixThreads / 32 ? red_m[lane] : -INFINITY;
            s = lane < kMixThreads / 32 ? red_s[lane] : 0.f;
            for (int o = 16; o > 0; o >>= 1) lse_merge(m, s, __shfl_xor_sync(0xffffffffu, m, o), __shfl_xor_sync(0xffffffffu, s, o));
            if (lane == 0) { row_m[k] = m; row_s[k] = s; }
        }
        __syncthreads();
    }
    float* o = out + (long)blockIdx.x * ld_out;
    for (int v = threadIdx.x; v < V1; v += kMixThreads) {
        float acc = 0.f;
        for (int k = 0; k < mw.K; ++k) acc += expf(zr[k * member_stride + v] - row_m[k]) / row_s[k] * mw.w[k] / mw.sum;
        o[v] = logf(acc);
    }
}

namespace {

int mix_launch(const float* z, long member_stride, int rows, int V1, const MixWeights& mw, float* out, long ld_out, cudaStream_t st) {
    if (rows <= 0) return 0;
    capb_ensemble_mix_kernel<<<rows, kMixThreads, 0, st>>>(z, member_stride, V1, mw, out, ld_out);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

struct Member {
    EngineBase* e = nullptr;
    int R = 1;                 // region count the member runs with (1 for NewFC, which reads the fc features only)
};

struct Members {
    Member m[CAPB200_ENSEMBLE_MAX_MEMBERS];
    int K = 0;
    MixWeights mw{};
};

// Everything the reference takes from models[0] or that would make the mixture meaningless is refused here, before any device work.
int resolve(const capb200_ensemble_member* members, int K, const float* fc, const float* att, int R, Members& E) {
    CAPB_REQUIRE(members != nullptr && K >= 1 && K <= CAPB200_ENSEMBLE_MAX_MEMBERS, "an ensemble has 1..8 members");
    E.K = K;
    E.mw.K = K;
    float sum = 0.f;
    for (int k = 0; k < K; ++k) {
        const capb200_ensemble_member& c = members[k];
        CAPB_REQUIRE(std::isfinite(c.weight) && c.weight >= 0.f, "ensemble weights must be finite and >= 0");
        CAPB_REQUIRE(c.engine != nullptr, "null member engine");
        CAPB_REQUIRE(c.family == CAPB200_FAMILY_UPDOWN || c.family == CAPB200_FAMILY_NEWFC || c.family == CAPB200_FAMILY_ATT2IN2 ||
                     c.family == CAPB200_FAMILY_AOA, "ensemble members are UpDown, NewFC, Att2in2 or AoANet engines");
        E.mw.w[k] = c.weight;
        sum += c.weight;
    }
    CAPB_REQUIRE(sum > 0.f, "ensemble weights must not all be zero");
    E.mw.sum = sum;
    bool reads_fc = false, reads_att = false;
    int dev = -1;
    CAPB_CHECK_CUDA(cudaGetDevice(&dev));
    for (int k = 0; k < K; ++k) {
        const capb200_ensemble_member& c = members[k];
        Member& m = E.m[k];
        // the handle's type is the one its declared family names (include/capb200.h: capb200_ensemble_member)
        m.e = c.family == CAPB200_FAMILY_AOA ? engine_base(static_cast<capb200_aoa_engine*>(c.engine)) : engine_base(static_cast<capb200_engine*>(c.engine));
        if (check_ready(m.e)) return 1;
        CAPB_REQUIRE(m.e->family == c.family, "member family does not match its engine");
        CAPB_REQUIRE(m.e->V1 == E.m[0].e->V1 && m.e->T == E.m[0].e->T, "every member needs the first member's vocab_size and seq_length (AttEnsemble.py:22-23)");
        cudaPointerAttributes pa;
        CAPB_CHECK_CUDA(cudaPointerGetAttributes(&pa, m.e->wblock));
        CAPB_REQUIRE(pa.device == dev, "every member must live on the current device");
        m.R = m.e->reads_att ? R : 1;
        reads_att |= m.e->reads_att;
        reads_fc |= m.e->reads_fc;
    }
    CAPB_REQUIRE(!reads_fc || fc != nullptr, "fc features required");
    CAPB_REQUIRE(!reads_att || (att != nullptr && R >= 1), "attention features required");
    return 0;
}

// the third extent of the ensemble's workspace is the caption length
int ensure_workspace(capb200_ensemble* s, int B, int rows, int beam, int T, cudaStream_t st) {
    return s->grow(B, rows, T, beam, st, [&](Arena& a, int nB, int nRows, int nT, int nBeam) { s->d.carve(a, nB, nRows, nBeam, nT); });
}

// Sizes every workspace for `rows` rows and runs each member's prologue; member launches are counted as the ensemble's.
int setup(capb200_ensemble* s, Members& E, const float* fc, const float* att, const float* mask, int B, int rows, int beam, int rows_per_image,
          cudaStream_t st) {
    const int V1 = E.m[0].e->V1, T = E.m[0].e->T;
    if (ensure_workspace(s, B, rows, beam, T, st)) return 1;
    if (grow_buffer(reinterpret_cast<void**>(&s->mix), &s->mix_bytes, sizeof(float) * E.K * rows * (size_t)V1, st)) return 1;
    for (int k = 0; k < E.K; ++k) {
        EngineBase* e = E.m[k].e;
        const long l0 = e->launches;
        const int rc = e->decode_workspace(B, rows, E.m[k].R, beam, rows_per_image, st) || e->decode_prepare(fc, att, {B, E.m[k].R, mask}, st);
        s->launches += e->launches - l0;
        if (rc) return 1;
    }
    return 0;
}

// One ensemble step on `rows` rows: every member's core into its slice of s->mix, then the mixture into `logits`.  A fresh state (the
// drivers pass their own all -1 table) is handed to each member as that member's fresh-state table: NewFC recognises it by address.
int step(capb200_ensemble* s, Members& E, int rows, int rpi, const int* tokens, const int* src_row, int t, float* logits, long ld, long member_stride,
         int B, const float* mask, cudaStream_t st) {
    const int V1 = E.m[0].e->V1;
    const bool fresh = src_row == s->d.neg1;
    for (int k = 0; k < E.K; ++k) {
        EngineBase* e = E.m[k].e;
        const long l0 = e->launches;
        const int rc = e->decode_core(rows, rpi, tokens, fresh ? e->d.neg1 : src_row, t, s->mix + k * member_stride, V1, {B, E.m[k].R, mask}, st);
        s->launches += e->launches - l0;
        if (rc) return 1;
    }
    s->launches++;
    return mix_launch(s->mix, member_stride, rows, V1, E.mw, logits, ld, st);
}

// Key of everything outside the beam driver that the captured loop depends on: the ensemble's buffers and, per member, its workspace, weight
// block, mask pointer, region count, family and weight (the weights are kernel arguments of the mixing launches).  0 disables the graph.
unsigned long long graph_key(const capb200_ensemble* s, const Members& E, const float* mask) {
    unsigned long long h = 1469598103934665603ull;
    auto mix = [&](unsigned long long v) { h ^= v; h *= 1099511628211ull; };
    mix(reinterpret_cast<uintptr_t>(s->ws)); mix(reinterpret_cast<uintptr_t>(s->mix)); mix((unsigned long long)E.K);
    for (int k = 0; k < E.K; ++k) {
        const Member& m = E.m[k];
        if (!m.e->loop_graph_ok()) return 0;
        unsigned bits = 0;
        memcpy(&bits, &E.mw.w[k], sizeof(float));
        mix(loop_graph_key(m.e->ws, m.e->wblock, mask, m.R, m.e->family));
        mix((unsigned long long)bits);
    }
    return h | 1ull;
}

}  // namespace
}  // namespace capb200

extern "C" {

capb200_ensemble* capb200_ensemble_create(void) { return new capb200_ensemble(); }

void capb200_ensemble_destroy(capb200_ensemble* s) {
    if (s == nullptr) return;
    if (s->ws != nullptr || s->mix != nullptr) {         // nothing to release on the device if it never decoded
        s->release();
        cudaFree(s->mix);
    }
    delete s;
}

long capb200_ensemble_launch_count(const capb200_ensemble* s) { return s ? s->launches : 0; }

int capb200_ensemble_decode_beam(capb200_ensemble* s, const capb200_ensemble_member* members, int K, const float* fc, const float* att,
                                 const float* mask, int B, int R, const capb200_beam_opts* opts, long long* seq, float* seq_logprobs,
                                 long long* done_seq, int* done_len, float* done_p, float* done_raw, void* stream) {
    CAPB_REQUIRE(s != nullptr, "null argument");
    Members E;
    if (resolve(members, K, fc, att, R, E)) return 1;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int V1 = E.m[0].e->V1, T = E.m[0].e->T;
    if (check_beam_opts(opts, V1, seq)) return 1;
    CAPB_REQUIRE(B >= 1, "empty batch");
    const int beam = opts->beam_size, keep = opts->sample_n;
    const int rows = B * beam;
    if (setup(s, E, fc, att, mask, B, rows, beam, 1, st)) return 1;
    s->V1 = V1; s->T = T;
    const long stride = (long)rows * V1;
    auto core = [&](int nrows, int live, const int* tokens, const int* src_row, int t, float* logits, long ld) {
        return step(s, E, nrows, live, tokens, src_row, t, logits, ld, stride, B, mask, st);
    };
    return beam_decode_driver(s->d, V1, T, B, beam, keep, opts->penalty_kind, opts->penalty_alpha, seq, seq_logprobs, done_seq, done_len, done_p,
                              done_raw, core, &s->launches, st, graph_key(s, E, mask), to_edits(opts->edits), opts->temperature);
}

int capb200_ensemble_beam_record_logprobs(capb200_ensemble* s, int image, int rank, float* dst, void* stream) {
    CAPB_REQUIRE(s != nullptr && dst != nullptr, "null argument");
    return beam_record_logprobs(s->d, s->V1, s->T, image, rank, dst, static_cast<cudaStream_t>(stream));
}

int capb200_ensemble_decode_sample(capb200_ensemble* s, const capb200_ensemble_member* members, int K, const float* fc, const float* att,
                                   const float* mask, int B, int R, const capb200_sample_opts* opts, const long long* tokens_in, long ld_tok,
                                   long long* seq, float* seq_logprobs, float* picked, void* stream) {
    CAPB_REQUIRE(s != nullptr, "null argument");
    Members E;
    if (resolve(members, K, fc, att, R, E)) return 1;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int V1 = E.m[0].e->V1, T = E.m[0].e->T;
    int steps = 0;
    if (check_sample_opts(opts, B, T, 1 << 30, tokens_in, ld_tok, seq, seq_logprobs, &steps)) return 1;
    const int n = opts->sample_n, rows = B * n;
    if (setup(s, E, fc, att, mask, B, rows, 1, n, st)) return 1;
    const long stride = (long)rows * V1;
    auto core = [&](int nrows, int /*live*/, const int* tokens, const int* src_row, int t, float* logits, long ld) {
        return step(s, E, nrows, n, tokens, src_row, t, logits, ld, stride, B, mask, st);
    };
    return sample_decode_driver(s->d, V1, T, rows, opts->method, opts->temperature, opts->seed, steps, tokens_in, ld_tok, seq, seq_logprobs, picked, core,
                                &s->launches, st, to_edits(opts->edits), opts->top);
}

}  // extern "C"
