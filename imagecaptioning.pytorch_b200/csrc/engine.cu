// Engine: owns packed weights + workspaces and drives the whole decode (prologue, T timesteps, beam bookkeeping) as a
// host-sync-free sequence of kernel launches on the caller's stream.  C ABI declared in include/capb200.h.
//
// Reference call stack this replaces (SURVEY.md section 3):
//   AttModel._sample_beam  AttModel.py:218-256  -> _prepare_feature :114-124, get_logprobs_state :166-176,
//                                                  CaptionModel.beam_search CaptionModel.py:35-209
//   AttModel._sample       AttModel.py:258-352  -> sample_next_word CaptionModel.py:370-407
//   AttModel._forward      AttModel.py:126-164
// Differences that matter for speed, none for results:
//   * image features (fc', att', p_att) are indexed per image, never replicated per beam (repeat_tensors, AttModel.py:241),
//   * the fc' contribution to the attention-LSTM gates is constant over time, so it is contracted once per image in the
//     prologue and enters every step as a per-image row bias (the reference re-multiplies it every step, AttModel.py:626),
//   * no per-step host synchronisation: EOS handling, finished-beam records and history live on the device.
#include <map>
#include <mutex>
#include <vector>

#include "../../include/capb200.h"
#include "common.cuh"
#include "kernels.cuh"
#include "engine_common.cuh"
#include "train_common.cuh"

namespace capb200 {

static thread_local std::string g_last_error;
void set_error(const std::string& msg) { g_last_error = msg; }
const char* last_error_cstr() { return g_last_error.c_str(); }

__global__ void capb_fill_int_kernel(int* p, int n, int v) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}
__global__ void capb_load_token_column_kernel(const long long* src, long ld, int col, int n, int* dst) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[i] = (int)src[(long)i * ld + col];
}
__global__ void capb_store_token_column_kernel(const int* src, int n, long long* dst, long ld, int col) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dst[(long)i * ld + col] = src[i];
}
int store_token_column_launch(const int* src, int n, long long* dst, long ld, int col, cudaStream_t st) {
    if (n <= 0) return 0;
    capb_store_token_column_kernel<<<cdiv(n, 256), 256, 0, st>>>(src, n, dst, ld, col);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}
int fill_int_launch(int* p, int n, int v, cudaStream_t st) {
    if (n <= 0) return 0;
    capb_fill_int_kernel<<<cdiv(n, 256), 256, 0, st>>>(p, n, v);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}
int load_token_column_launch(const long long* src, long ld, int col, int n, int* dst, cudaStream_t st) {
    if (n <= 0) return 0;
    capb_load_token_column_kernel<<<cdiv(n, 256), 256, 0, st>>>(src, ld, col, n, dst);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

namespace {

__global__ void add_vec_kernel(const float* a, const float* b, float* o, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) o[i] = a[i] + b[i];
}
__global__ void interleave_gates_kernel(const float* src, float* dst, int H) {      // dst[4*j+g] = src[g*H + j]
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < 4 * H) dst[i] = src[(i & 3) * H + (i >> 2)];
}

__global__ void iota_div_kernel(int* p, int n, int div) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = i / div;
}


enum GemmId { G_FC = 0, G_ATT, G_CTX, G_GFC, G_LSTM1, G_H2ATT, G_LSTM2, G_LOGIT, G_CORE, G_A2C, G_COUNT };
constexpr int G_REPORTED = 9;      // ids exposed through capb200_engine_read_profile (Att2in2's a2c launch is folded into G_CORE)

}  // namespace
}  // namespace capb200

using namespace capb200;


struct capb200_engine : EngineBase {
    capb200_model_cfg cfg{};
    capb200_weights w{};
    int E = 0, H = 0, A = 0;

    // bind-time buffers (in the weight block)
    float *bsum_att = nullptr, *bsum_lang = nullptr, *bsum_core = nullptr;
    float *bsum_att_il = nullptr, *bsum_lang_il = nullptr;   // gate-interleaved copies for the fused LSTM epilogue (tensor-core modes)
    float* xgate = nullptr;          // [V+1, 4H] relu(embed) * W_ih[:, 2H:]^T: per-token gate contribution (eval-mode decode)
    long ld_xgate = 0;
    bool use_xgate = true;
    Planes p_fc, p_attw, p_ctx, p_logit, p_a_ih_h, p_a_ih_fc, p_a_ih_x, p_a_hh, p_l_ih_a, p_l_ih_h, p_l_hh, p_h2att, p_i2h, p_h2h, p_a2c;

    // workspace
    Planes in_fc, in_att;                        // split copies of the user inputs (tensor-core modes)
    Act fc_e, att_e, p_att, g_fc, xt, h0_in, h1_in, h0_out, h1_out, att_res, att_h, gates;
    float *c0[2] = {nullptr, nullptr}, *c1[2] = {nullptr, nullptr};
    long ld_c = 0;
    int* img_of_row = nullptr;
    float* att_score = nullptr;   // [rows, R] attention scores
    int core_cur = 0;   // which c buffer currently holds the state

    // optional per-GEMM device timing (cudaEvent pairs on the launching stream), off by default
    bool profiling = false;
    std::vector<cudaEvent_t> ev_pool;
    std::vector<int> ev_ids;          // GEMM id of each recorded pair
    std::vector<double> ev_flops;     // algorithmic FLOPs of each recorded launch
    size_t ev_used = 0;
    double prof_ms[G_COUNT] = {0};
    double prof_flops[G_COUNT] = {0};
    long prof_calls[G_COUNT] = {0};

    ~capb200_engine() override { for (cudaEvent_t ev : ev_pool) cudaEventDestroy(ev); }
    int decode_workspace(int B, int rows, int R, int beam, int rows_per_image, cudaStream_t st) override;
    int decode_prepare(const float* fc, const float* att, const DecodeCtx& c, cudaStream_t st) override;
    int decode_core(int rows, int rpi, const int* tokens, const int* src_row, int t, float* logits, long ld, const DecodeCtx& c, cudaStream_t st) override;
    bool next_state(NextStateGather* next) override;
    bool loop_graph_ok() const override { return !profiling; }
};

namespace {

void layout_weights(capb200_engine* e, Arena& a) {
    const int H = e->H, E = e->E, A = e->A, V1 = e->V1;
    const bool updown = e->cfg.family == CAPB200_FAMILY_UPDOWN;
    e->bsum_att = a.take<float>(4 * H);
    e->bsum_lang = a.take<float>(4 * H);
    e->bsum_core = a.take<float>(5 * H);
    e->bsum_att_il = a.take<float>(4 * H);
    e->bsum_lang_il = a.take<float>(4 * H);
    if (updown) { e->ld_xgate = round_up(4 * H, 8); e->xgate = a.take<float>((long)V1 * e->ld_xgate); }
    if (!e->tc) return;
    e->p_logit = carve_planes(a, V1, H);
    if (updown) {
        e->p_fc = carve_planes(a, H, e->cfg.fc_feat_size);
        e->p_attw = carve_planes(a, H, e->cfg.att_feat_size);
        e->p_ctx = carve_planes(a, A, H);
        e->p_a_ih_h = carve_planes(a, 4 * H, H);
        e->p_a_ih_fc = carve_planes(a, 4 * H, H);
        e->p_a_ih_x = carve_planes(a, 4 * H, E);
        e->p_a_hh = carve_planes(a, 4 * H, H);
        e->p_l_ih_a = carve_planes(a, 4 * H, H);
        e->p_l_ih_h = carve_planes(a, 4 * H, H);
        e->p_l_hh = carve_planes(a, 4 * H, H);
        e->p_h2att = carve_planes(a, A, H);
    } else if (e->cfg.family == CAPB200_FAMILY_ATT2IN2) {
        e->p_attw = carve_planes(a, H, e->cfg.att_feat_size);
        e->p_ctx = carve_planes(a, A, H);
        e->p_h2att = carve_planes(a, A, H);
        e->p_i2h = carve_planes(a, 5 * H, E);
        e->p_h2h = carve_planes(a, 5 * H, H);
        e->p_a2c = carve_planes(a, 2 * H, H);
    } else {
        e->p_fc = carve_planes(a, E, e->cfg.fc_feat_size);
        e->p_i2h = carve_planes(a, 5 * H, E);
        e->p_h2h = carve_planes(a, 5 * H, H);
    }
}

void layout_workspace(capb200_engine* e, Arena& a, int B, int rows, int R, int beam) {
    const int H = e->H, E = e->E, A = e->A, T = e->T;
    const bool updown = e->cfg.family == CAPB200_FAMILY_UPDOWN;
    const bool attn = e->reads_att;
    const bool tc = e->tc;
    if (tc) {
        e->in_fc = carve_planes(a, B, e->cfg.fc_feat_size);
        if (attn) e->in_att = carve_planes(a, (long)B * R, e->cfg.att_feat_size);
    }
    e->fc_e.carve(a, B, updown ? H : E, tc);
    if (attn) {
        e->att_e.carve(a, (long)B * R, H, tc);
        e->p_att.carve(a, (long)B * R, A, false);
        e->att_res.carve(a, rows, H, tc);
        e->att_h.carve(a, rows, A, false);
    }
    if (updown) {
        e->g_fc.carve(a, B, 4 * H, false);
        e->h1_in.carve(a, rows, H, tc);
        e->h1_out.carve(a, rows, H, tc);
    }
    e->xt.carve(a, rows, E, tc);
    e->h0_in.carve(a, rows, H, tc);
    e->h0_out.carve(a, rows, H, tc);
    e->gates.carve(a, rows, 5 * H, false);
    e->ld_c = round_up(H, 8);
    for (int i = 0; i < 2; ++i) {
        e->c0[i] = a.take<float>((long)rows * e->ld_c);
        e->c1[i] = a.take<float>((long)rows * e->ld_c);
    }
    e->carve_head(a, rows);
    e->img_of_row = a.take<int>(rows);
    e->att_score = a.take<float>((long)rows * (R > 0 ? R : 1));
    e->d.carve(a, B, rows, beam, T);
}

int ensure_workspace(capb200_engine* e, int B, int rows, int R, int beam, cudaStream_t st) {
    return e->grow(B, rows, R, beam, st, [&](Arena& a, int nB, int nRows, int nR, int nBeam) { layout_workspace(e, a, nB, nRows, nR, nBeam); });
}

// ---- GEMM dispatch: the engine's GEMM, timed per launch while profiling ----------------------------------------------------------------------
int run_gemm(capb200_engine* e, int id, GemmProblem& g, int plan_rows, cudaStream_t st) {
    if (!e->profiling) return e->gemm(id, g, plan_rows, st);
    if (e->ev_used + 2 > e->ev_pool.size()) {
        for (int i = 0; i < 64; ++i) {
            cudaEvent_t ev;
            CAPB_CHECK_CUDA(cudaEventCreate(&ev));
            e->ev_pool.push_back(ev);
        }
    }
    double k_total = 0;
    for (int s = 0; s < g.nseg; ++s) k_total += g.seg[s].K;
    CAPB_CHECK_CUDA(cudaEventRecord(e->ev_pool[e->ev_used], st));
    const int rc = e->gemm(id, g, plan_rows, st);
    CAPB_CHECK_CUDA(cudaEventRecord(e->ev_pool[e->ev_used + 1], st));
    e->ev_used += 2;
    e->ev_ids.push_back(id);
    e->ev_flops.push_back(2.0 * g.M * g.N * k_total);
    return rc;
}

// ---- prologue: _prepare_feature ---------------------------------------------------------------------------------------
int prepare(capb200_engine* e, const float* fc, const float* att, const float* mask, int B, int R, cudaStream_t st) {
    CAPB_NVTX("capb200 prepare_feature (fc_embed, att_embed, ctx2att)");
    const int H = e->H, E = e->E, A = e->A;
    const bool updown = e->cfg.family == CAPB200_FAMILY_UPDOWN;
    const capb200_weights& w = e->w;
    ActView fc_in;  fc_in.f = const_cast<float*>(fc);  fc_in.ld = e->cfg.fc_feat_size;
    if (e->tc && e->cfg.family != CAPB200_FAMILY_ATT2IN2) {
        e->launches++;
        if (split_planes_launch(fc, e->cfg.fc_feat_size, B, e->cfg.fc_feat_size, e->in_fc.hi, e->in_fc.lo, e->in_fc.ld, st)) return 1;
    }
    if (e->cfg.family != CAPB200_FAMILY_ATT2IN2) {   // fc_embed: Linear (+ReLU for UpDown; NewFC has a bare Linear, AttModel.py:907; Att2in2 has none, :858)
        GemmProblem g;
        g.M = B; g.N = updown ? H : E; g.nseg = 1;
        g.seg[0] = seg_of(fc_in, w.fc_embed_w, e->cfg.fc_feat_size, e->p_fc, e->cfg.fc_feat_size);
        g.seg[0].A_hi = e->in_fc.hi; g.seg[0].A_lo = e->in_fc.lo; g.seg[0].lda_h = e->in_fc.ld;
        g.epi.bias = w.fc_embed_b; g.epi.relu = updown ? 1 : 0;
        g.epi.C = e->fc_e.v.f; g.epi.ldc = e->fc_e.v.ld; g.epi.C_hi = e->fc_e.v.hi; g.epi.C_lo = e->fc_e.v.lo; g.epi.ldcs = e->fc_e.v.ld;
        if (run_gemm(e, G_FC, g, e->capB, st)) return 1;
    }
    if (!e->reads_att) return 0;
    ActView att_in; att_in.f = const_cast<float*>(att); att_in.ld = e->cfg.att_feat_size;
    if (e->tc) {
        e->launches++;
        if (split_planes_launch(att, e->cfg.att_feat_size, B * R, e->cfg.att_feat_size, e->in_att.hi, e->in_att.lo, e->in_att.ld, st)) return 1;
    }
    {   // att_embed: the one consumer of the [B,R,2048] bottom-up tile (AttModel.py:119)
        GemmProblem g;
        g.M = B * R; g.N = H; g.nseg = 1;
        g.seg[0] = seg_of(att_in, w.att_embed_w, e->cfg.att_feat_size, e->p_attw, e->cfg.att_feat_size);
        g.seg[0].A_hi = e->in_att.hi; g.seg[0].A_lo = e->in_att.lo; g.seg[0].lda_h = e->in_att.ld;
        g.epi.bias = w.att_embed_b; g.epi.relu = 1;
        g.epi.C = e->att_e.v.f; g.epi.ldc = e->att_e.v.ld; g.epi.C_hi = e->att_e.v.hi; g.epi.C_lo = e->att_e.v.lo; g.epi.ldcs = e->att_e.v.ld;
        if (run_gemm(e, G_ATT, g, e->capB * e->capR, st)) return 1;
    }
    if (mask != nullptr) {   // pack_wrapper zero-pads the rows of invalid regions (AttModel.py:44-49)
        e->launches++;
        if (mask_rows_launch(e->att_e.v, B, R, H, mask, R, st)) return 1;
    }
    {   // ctx2att
        GemmProblem g;
        g.M = B * R; g.N = A; g.nseg = 1;
        g.seg[0] = seg_of(e->att_e.v, w.ctx2att_w, H, e->p_ctx, H);
        g.epi.bias = w.ctx2att_b;
        g.epi.C = e->p_att.v.f; g.epi.ldc = e->p_att.v.ld;
        if (run_gemm(e, G_CTX, g, e->capB * e->capR, st)) return 1;
    }
    if (!updown) return 0;
    {   // time-invariant part of the attention-LSTM gates: fc' * W_ih[:, H:2H]^T + b_ih + b_hh
        GemmProblem g;
        g.M = B; g.N = 4 * H; g.nseg = 1;
        g.seg[0] = seg_of(e->fc_e.v, w.att_lstm_w_ih + H, E + 2 * H, e->p_a_ih_fc, H);
        g.epi.bias = e->tc ? e->bsum_att_il : e->bsum_att;     // tensor-core modes keep every gate quantity interleaved
        g.epi.C = e->g_fc.v.f; g.epi.ldc = e->g_fc.v.ld;
        if (run_gemm(e, G_GFC, g, e->capB, st)) return 1;
    }
    return 0;
}

// ---- the vocabulary projection of the core's output `h` (through the logit head's hidden layers, if any) into the caller's log-prob storage
int logit_gemm(capb200_engine* e, const ActView& h, int rows, float* logits, long ld_logits, cudaStream_t st) {
    ActView x;
    if (e->run_logit_head(h, rows, &x, st)) return 1;
    GemmProblem g;
    g.M = rows; g.N = e->V1; g.nseg = 1;
    g.seg[0] = seg_of(x, e->w.logit_w, e->H, e->p_logit, e->H);
    g.epi.bias = e->w.logit_b;
    g.epi.C = logits; g.epi.ldc = ld_logits;
    return run_gemm(e, G_LOGIT, g, e->capRows, st);
}

// ---- one application of the recurrent core on `rows` rows (rpi rows per image) -----------------------------------------
// tokens: input word per row; src_row: parent row per row (nullptr = identity, e->neg1 = fresh zero state)
// states_gathered (UpDown): h0_in / h1_in already hold the parents' states (the previous step's beam_search_step_kernel wrote them)
int core_step(capb200_engine* e, int rows, int rpi, const int* tokens, const int* src_row, float* logits, long ld_logits, int n_images, int R,
              const float* mask, cudaStream_t st, bool states_gathered = false) {
    const int H = e->H, E = e->E, A = e->A;
    const capb200_weights& w = e->w;
    if (e->cfg.family == CAPB200_FAMILY_UPDOWN) {
        StateCopy s0, s1;
        s0.src = e->h0_out.v.f; s0.ld_src = e->h0_out.v.ld; s0.dst = e->h0_in.v;
        s1.src = e->h1_out.v.f; s1.ld_src = e->h1_out.v.ld; s1.dst = e->h1_in.v;
        const bool xg = e->use_xgate;     // word contribution comes from the per-token table instead of a K-segment
        CAPB_REQUIRE(!states_gathered || xg, "the fused beam step gathers the states only; the word embedding needs the separate gather");
        if (!states_gathered) {
            e->launches++;
            if (state_gather_embed_launch(rows, tokens, src_row, w.embed, E, xg ? 0 : E, 1, e->xt.v, H, 2, s0, s1, st)) return 1;
        }
        const int cur = e->core_cur, nxt = cur ^ 1;
        {   // attention LSTM gates: [h_lang_prev | (xt) | h_att_prev] segments + per-image fc' term
            GemmProblem g;
            g.M = rows; g.N = 4 * H;
            g.seg[0] = seg_of(e->h1_in.v, w.att_lstm_w_ih, E + 2 * H, e->p_a_ih_h, H);
            g.seg[1] = seg_of(e->h0_in.v, w.att_lstm_w_hh, H, e->p_a_hh, H);
            g.nseg = 2;
            if (!xg) { g.seg[2] = seg_of(e->xt.v, w.att_lstm_w_ih + 2 * H, E + 2 * H, e->p_a_ih_x, E); g.nseg = 3; }
            g.epi.row_bias = e->g_fc.v.f; g.epi.ld_row_bias = e->g_fc.v.ld; g.epi.rows_per_group = rpi;
            if (e->tc) {     // cell applied in the GEMM epilogue: no gate buffer, no point-wise launch
                g.epi.lstm = 1; g.epi.H = H;
                g.epi.c_prev = e->c0[cur]; g.epi.ld_cprev = e->ld_c; g.epi.src_row = src_row;
                g.epi.c_out = e->c0[nxt]; g.epi.ld_cout = e->ld_c;
                g.epi.gather_bias = xg ? e->xgate : nullptr; g.epi.ld_gb = e->ld_xgate; g.epi.gather_idx = tokens;
                g.epi.h_f = e->h0_out.v.f; g.epi.h_hi = e->h0_out.v.hi; g.epi.h_lo = e->h0_out.v.lo; g.epi.ld_h = e->h0_out.v.ld;
            } else {
                g.epi.C = e->gates.v.f; g.epi.ldc = e->gates.v.ld;
            }
            if (run_gemm(e, G_LSTM1, g, e->capRows, st)) return 1;
        }
        if (!e->tc) {
            e->launches++;
            if (lstm_pointwise_launch(rows, H, e->gates.v.f, e->gates.v.ld, src_row, e->c0[cur], e->ld_c, e->c0[nxt], e->ld_c, e->h0_out.v,
                                      xg ? e->xgate : nullptr, e->ld_xgate, tokens, st)) return 1;
        }
        {   // h2att
            GemmProblem g;
            g.M = rows; g.N = A; g.nseg = 1;
            g.seg[0] = seg_of(e->h0_out.v, w.h2att_w, H, e->p_h2att, H);
            g.epi.bias = w.h2att_b;
            g.epi.C = e->att_h.v.f; g.epi.ldc = e->att_h.v.ld;
            if (run_gemm(e, G_H2ATT, g, e->capRows, st)) return 1;
        }
        e->launches += 2;
        if (additive_attention_launch(n_images, rpi, R, A, H, e->att_h.v.f, e->att_h.v.ld, e->p_att.v.f, e->p_att.v.ld, e->att_e.v.f, e->att_e.v.ld,
                                      mask, R, w.alpha_w, w.alpha_b, e->att_score, e->att_res.v, st)) return 1;
        {   // language LSTM gates: [att_res | h_att | h_lang_prev]
            GemmProblem g;
            g.M = rows; g.N = 4 * H; g.nseg = 3;
            g.seg[0] = seg_of(e->att_res.v, w.lang_lstm_w_ih, 2 * H, e->p_l_ih_a, H);
            g.seg[1] = seg_of(e->h0_out.v, w.lang_lstm_w_ih + H, 2 * H, e->p_l_ih_h, H);
            g.seg[2] = seg_of(e->h1_in.v, w.lang_lstm_w_hh, H, e->p_l_hh, H);
            if (e->tc) {
                g.epi.bias = e->bsum_lang_il;
                g.epi.lstm = 1; g.epi.H = H;
                g.epi.c_prev = e->c1[cur]; g.epi.ld_cprev = e->ld_c; g.epi.src_row = src_row;
                g.epi.c_out = e->c1[nxt]; g.epi.ld_cout = e->ld_c;
                g.epi.h_f = e->h1_out.v.f; g.epi.h_hi = e->h1_out.v.hi; g.epi.h_lo = e->h1_out.v.lo; g.epi.ld_h = e->h1_out.v.ld;
            } else {
                g.epi.bias = e->bsum_lang;
                g.epi.C = e->gates.v.f; g.epi.ldc = e->gates.v.ld;
            }
            if (run_gemm(e, G_LSTM2, g, e->capRows, st)) return 1;
        }
        if (!e->tc) {
            e->launches++;
            if (lstm_pointwise_launch(rows, H, e->gates.v.f, e->gates.v.ld, src_row, e->c1[cur], e->ld_c, e->c1[nxt], e->ld_c, e->h1_out.v,
                                      nullptr, 0, nullptr, st)) return 1;
        }
        e->core_cur = nxt;
        return logit_gemm(e, e->h1_out.v, rows, logits, ld_logits, st);
    }
    if (e->cfg.family == CAPB200_FAMILY_ATT2IN2) {
        // ---- Att2in2 (AttModel.py:770-790): attention on the PREVIOUS h, maxout cell whose candidate pair also gets a2c(att_res).
        // A fresh row (src_row < 0) gathers h = 0, so its att_h is the h2att bias and the cell sees c = 0.
        StateCopy s0, s1;
        s0.src = e->h0_out.v.f; s0.ld_src = e->h0_out.v.ld; s0.dst = e->h0_in.v;
        e->launches++;
        if (state_gather_embed_launch(rows, tokens, src_row, w.embed, E, E, 1, e->xt.v, H, 1, s0, s1, st)) return 1;
        const int cur = e->core_cur, nxt = cur ^ 1;
        {   // h2att on h_prev
            GemmProblem g;
            g.M = rows; g.N = A; g.nseg = 1;
            g.seg[0] = seg_of(e->h0_in.v, w.h2att_w, H, e->p_h2att, H);
            g.epi.bias = w.h2att_b;
            g.epi.C = e->att_h.v.f; g.epi.ldc = e->att_h.v.ld;
            if (run_gemm(e, G_H2ATT, g, e->capRows, st)) return 1;
        }
        e->launches += 2;
        if (additive_attention_launch(n_images, rpi, R, A, H, e->att_h.v.f, e->att_h.v.ld, e->p_att.v.f, e->p_att.v.ld, e->att_e.v.f, e->att_e.v.ld,
                                      mask, R, w.alpha_w, w.alpha_b, e->att_score, e->att_res.v, st)) return 1;
        {   // sums = [xt | h_prev] [i2h | h2h]^T + (i2h_b + h2h_b + [0 | a2c_b])
            GemmProblem g;
            g.M = rows; g.N = 5 * H; g.nseg = 2;
            g.seg[0] = seg_of(e->xt.v, w.i2h_w, E, e->p_i2h, E);
            g.seg[1] = seg_of(e->h0_in.v, w.h2h_w, H, e->p_h2h, H);
            g.epi.bias = e->bsum_core;
            g.epi.C = e->gates.v.f; g.epi.ldc = e->gates.v.ld;
            if (run_gemm(e, G_CORE, g, e->capRows, st)) return 1;
        }
        {   // sums[:, 3H:5H] += att_res a2c^T  (in place through the residual epilogue)
            GemmProblem g;
            g.M = rows; g.N = 2 * H; g.nseg = 1;
            g.seg[0] = seg_of(e->att_res.v, w.a2c_w, H, e->p_a2c, H);
            g.epi.residual = e->gates.v.f + 3 * H; g.epi.ld_res = e->gates.v.ld;
            g.epi.C = e->gates.v.f + 3 * H; g.epi.ldc = e->gates.v.ld;
            if (run_gemm(e, G_A2C, g, e->capRows, st)) return 1;
        }
        e->launches++;
        if (maxout_pointwise_launch(rows, H, e->gates.v.f, e->gates.v.ld, src_row, e->c0[cur], e->ld_c, e->c0[nxt], e->ld_c, e->h0_out.v, st)) return 1;
        e->core_cur = nxt;
        return logit_gemm(e, e->h0_out.v, rows, logits, ld_logits, st);
    }
    // ---- NewFC: maxout LSTM; a fresh state first consumes the image embedding (AttModel.py:925-936)
    const bool fresh = (src_row == e->d.neg1);
    for (int pass = fresh ? 0 : 1; pass < 2; ++pass) {
        StateCopy s0, s1;
        s0.src = e->h0_out.v.f; s0.ld_src = e->h0_out.v.ld; s0.dst = e->h0_in.v;
        const int* srcs = (pass == 0) ? e->d.neg1 : (fresh ? nullptr : src_row);
        e->launches++;
        if (pass == 0) {
            if (state_gather_embed_launch(rows, e->img_of_row, srcs, e->fc_e.v.f, e->fc_e.v.ld, E, 0, e->xt.v, H, 1, s0, s1, st)) return 1;
        } else {
            if (state_gather_embed_launch(rows, tokens, srcs, w.embed, E, E, 0, e->xt.v, H, 1, s0, s1, st)) return 1;
        }
        const int cur = e->core_cur, nxt = cur ^ 1;
        GemmProblem g;
        g.M = rows; g.N = 5 * H; g.nseg = 2;
        g.seg[0] = seg_of(e->xt.v, w.i2h_w, E, e->p_i2h, E);
        g.seg[1] = seg_of(e->h0_in.v, w.h2h_w, H, e->p_h2h, H);
        g.epi.bias = e->bsum_core;
        g.epi.C = e->gates.v.f; g.epi.ldc = e->gates.v.ld;
        if (run_gemm(e, G_CORE, g, e->capRows, st)) return 1;
        e->launches++;
        if (maxout_pointwise_launch(rows, H, e->gates.v.f, e->gates.v.ld, srcs, e->c0[cur], e->ld_c, e->c0[nxt], e->ld_c, e->h0_out.v, st)) return 1;
        e->core_cur = nxt;
    }
    return logit_gemm(e, e->h0_out.v, rows, logits, ld_logits, st);
}

}  // namespace

// ---- pieces the AoA engine shares (engine_common.cuh) and the decode hooks ------------------------------------------------------------------
namespace capb200 {

int add_vec_launch(const float* a, const float* b, float* o, int n, cudaStream_t st) {
    add_vec_kernel<<<cdiv(n, 256), 256, 0, st>>>(a, b, o, n);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int interleave_gates_launch(const float* src, float* dst, int H, cudaStream_t st) {
    interleave_gates_kernel<<<cdiv(4 * H, 256), 256, 0, st>>>(src, dst, H);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int build_gate_table(EngineBase& e, const float* embed, int E, int H, const float* w_x, long ld_w, const Planes& p_x, float* xgate, long ld_xgate,
                     cudaStream_t st) {
    const int V1 = e.V1;
    const long ldE = round_up(E, 8);
    char* tmp = nullptr;
    const size_t tmp_bytes = (size_t)V1 * ldE * (sizeof(float) + (e.tc ? 2 * sizeof(__half) : 0)) + 1024;
    CAPB_CHECK_CUDA(cudaMallocAsync(&tmp, tmp_bytes, st));
    CAPB_CHECK_CUDA(cudaMemsetAsync(tmp, 0, tmp_bytes, st));
    ActView ev;
    ev.ld = ldE;
    ev.f = reinterpret_cast<float*>(tmp);
    if (e.tc) {
        ev.hi = reinterpret_cast<__half*>(tmp + (size_t)V1 * ldE * sizeof(float));
        ev.lo = ev.hi + (size_t)V1 * ldE;
    }
    int rc = 0;
    if (ldE == E) {
        rc = relu_copy_launch(embed, (long)V1 * E, ev, st);
    } else {
        for (int v = 0; v < V1 && !rc; ++v) {     // ragged pitch (tiny test configs only): row by row
            ActView rv = ev;
            rv.f += (long)v * ldE; if (rv.hi) { rv.hi += (long)v * ldE; rv.lo += (long)v * ldE; }
            rc = relu_copy_launch(embed + (long)v * E, E, rv, st);
        }
    }
    GemmProblem g;
    g.M = V1; g.N = 4 * H; g.nseg = 1;
    g.seg[0] = seg_of(ev, w_x, ld_w, p_x, E);
    g.epi.C = xgate; g.epi.ldc = ld_xgate;
    if (!rc) {
        if (!e.tc) {
            rc = gemm_simt_launch(g, st);
        } else {
            GemmTcPlan* plan = gemm_tc_plan_create(g, e.mode == CAPB200_MODE_TC_F16X3 ? 3 : 1);
            rc = plan ? gemm_tc_plan_launch(plan, nullptr, 0, st) : 1;
            if (plan) gemm_tc_plan_destroy(plan);
        }
    }
    e.launches += 2;
    cudaFreeAsync(tmp, st);
    return rc;
}

EngineBase* engine_base(capb200_engine* e) { return e; }

}  // namespace capb200

int capb200_engine::decode_workspace(int B, int rows, int R, int beam, int rows_per_image, cudaStream_t st) {
    if (ensure_workspace(this, B, rows, R, beam, st)) return 1;
    if (!reads_att) { iota_div_kernel<<<cdiv(rows, 256), 256, 0, st>>>(img_of_row, rows, rows_per_image); launches++; }
    return 0;
}

int capb200_engine::decode_prepare(const float* fc, const float* att, const DecodeCtx& c, cudaStream_t st) {
    if (prepare(this, fc, att, c.mask, c.B, c.R, st)) return 1;
    core_cur = 0;
    return 0;
}

int capb200_engine::decode_core(int rows, int rpi, const int* tokens, const int* src_row, int /*t*/, float* logits, long ld, const DecodeCtx& c,
                                cudaStream_t st) {
    return core_step(this, rows, rpi, tokens, src_row, logits, ld, c.B, c.R, c.mask, st, d.states_gathered);
}

// UpDown's two states can be gathered by the fused beam step (the word enters through the per-token gate table, not an embedding copy)
bool capb200_engine::next_state(NextStateGather* next) {
    if (cfg.family != CAPB200_FAMILY_UPDOWN || !use_xgate) return false;
    next->s0.src = h0_out.v.f; next->s0.ld_src = h0_out.v.ld; next->s0.dst = h0_in.v;
    next->s1.src = h1_out.v.f; next->s1.ld_src = h1_out.v.ld; next->s1.dst = h1_in.v;
    next->H = H;
    return true;
}

// =====================================================================================================================
// C ABI
// =====================================================================================================================
extern "C" {

const char* capb200_last_error(void) { return g_last_error.c_str(); }
int capb200_abi_version(void) { return CAPB200_ABI_VERSION; }
int capb200_range_status(int reset) { return range_flag_read(reset); }

capb200_engine* capb200_engine_create(const capb200_model_cfg* cfg) {
    if (cfg == nullptr) { set_error("null cfg"); return nullptr; }
    if (cfg->family != CAPB200_FAMILY_UPDOWN && cfg->family != CAPB200_FAMILY_NEWFC && cfg->family != CAPB200_FAMILY_ATT2IN2) {
        set_error("unknown model family");
        return nullptr;
    }
    capb200_engine* e = create_engine<capb200_engine>(cfg->vocab_size, cfg->seq_length, cfg->numeric_mode, G_COUNT);
    if (e == nullptr) return nullptr;
    e->cfg = *cfg;
    e->E = cfg->input_encoding_size;
    e->H = cfg->rnn_size;
    e->A = cfg->att_hid_size;
    e->bind_name = "capb200_engine_bind_weights";
    e->family = e->graph_family = cfg->family;
    e->reads_fc = cfg->family != CAPB200_FAMILY_ATT2IN2;
    e->reads_att = cfg->family != CAPB200_FAMILY_NEWFC;
    return e;
}

void capb200_engine_destroy(capb200_engine* e) { delete e; }

long capb200_engine_launch_count(const capb200_engine* e) { return e ? e->launches : 0; }

int capb200_engine_set_profiling(capb200_engine* e, int enable) {
    CAPB_REQUIRE(e != nullptr, "null engine");
    e->profiling = enable != 0;
    return 0;
}

int capb200_engine_read_profile(capb200_engine* e, int reset, double* ms, double* flops, long* calls, int n) {
    CAPB_REQUIRE(e != nullptr && n >= G_REPORTED, "need room for 9 GEMM ids");
    CAPB_CHECK_CUDA(cudaDeviceSynchronize());
    for (size_t i = 0; i < e->ev_ids.size(); ++i) {
        float t = 0.f;
        CAPB_CHECK_CUDA(cudaEventElapsedTime(&t, e->ev_pool[2 * i], e->ev_pool[2 * i + 1]));
        e->prof_ms[e->ev_ids[i]] += t;
        e->prof_flops[e->ev_ids[i]] += e->ev_flops[i];
        e->prof_calls[e->ev_ids[i]] += 1;
    }
    e->ev_ids.clear();
    e->ev_flops.clear();
    e->ev_used = 0;
    // Att2in2's a2c launch reports under the core id
    e->prof_ms[G_CORE] += e->prof_ms[G_A2C]; e->prof_flops[G_CORE] += e->prof_flops[G_A2C]; e->prof_calls[G_CORE] += e->prof_calls[G_A2C];
    e->prof_ms[G_A2C] = 0; e->prof_flops[G_A2C] = 0; e->prof_calls[G_A2C] = 0;
    for (int i = 0; i < G_REPORTED; ++i) {
        if (ms) ms[i] = e->prof_ms[i];
        if (flops) flops[i] = e->prof_flops[i];
        if (calls) calls[i] = e->prof_calls[i];
        if (reset) { e->prof_ms[i] = 0; e->prof_flops[i] = 0; e->prof_calls[i] = 0; }
    }
    return 0;
}

int capb200_engine_bind_weights(capb200_engine* e, const capb200_weights* w, void* stream) {
    CAPB_REQUIRE(e != nullptr && w != nullptr, "null argument");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool updown = e->cfg.family == CAPB200_FAMILY_UPDOWN;
    const bool att2in2 = e->cfg.family == CAPB200_FAMILY_ATT2IN2;
    CAPB_REQUIRE(w->embed && (att2in2 || (w->fc_embed_w && w->fc_embed_b)) && w->logit_w && w->logit_b, "missing shared weights");
    if (att2in2) {
        CAPB_REQUIRE(w->att_embed_w && w->att_embed_b && w->ctx2att_w && w->ctx2att_b && w->h2att_w && w->h2att_b && w->alpha_w && w->alpha_b &&
                         w->i2h_w && w->i2h_b && w->h2h_w && w->h2h_b && w->a2c_w && w->a2c_b, "missing Att2in2 weights");
    } else if (updown) {
        CAPB_REQUIRE(w->att_embed_w && w->att_embed_b && w->ctx2att_w && w->ctx2att_b && w->att_lstm_w_ih && w->att_lstm_w_hh && w->att_lstm_b_ih &&
                         w->att_lstm_b_hh && w->lang_lstm_w_ih && w->lang_lstm_w_hh && w->lang_lstm_b_ih && w->lang_lstm_b_hh && w->h2att_w &&
                         w->h2att_b && w->alpha_w && w->alpha_b, "missing UpDown weights");
    } else {
        CAPB_REQUIRE(w->i2h_w && w->i2h_b && w->h2h_w && w->h2h_b, "missing NewFC weights");
    }
    e->w = *w;
    const int H = e->H, E = e->E, A = e->A, V1 = e->V1;
    if (e->alloc_wblock(st, [&](Arena& a) { layout_weights(e, a); })) return 1;
    int rc = 0;
    if (updown) {
        rc |= add_vec_launch(w->att_lstm_b_ih, w->att_lstm_b_hh, e->bsum_att, 4 * H, st);
        rc |= add_vec_launch(w->lang_lstm_b_ih, w->lang_lstm_b_hh, e->bsum_lang, 4 * H, st);
        rc |= interleave_gates_launch(e->bsum_att, e->bsum_att_il, H, st);
        rc |= interleave_gates_launch(e->bsum_lang, e->bsum_lang_il, H, st);
        e->launches += 4;
    } else {
        rc |= add_vec_launch(w->i2h_b, w->h2h_b, e->bsum_core, 5 * H, st);
        e->launches += 1;
        if (att2in2) {     // the a2c bias joins the candidate columns' bias: the a2c GEMM then needs no bias of its own
            rc |= add_vec_launch(e->bsum_core + 3 * H, w->a2c_b, e->bsum_core + 3 * H, 2 * H, st);
            e->launches += 1;
        }
    }
    if (rc) return 1;
    if (e->tc) {
        rc = e->pack(w->logit_w, H, V1, H, e->p_logit, st);
        if (updown) {
            rc |= e->pack(w->fc_embed_w, e->cfg.fc_feat_size, H, e->cfg.fc_feat_size, e->p_fc, st);
            rc |= e->pack(w->att_embed_w, e->cfg.att_feat_size, H, e->cfg.att_feat_size, e->p_attw, st);
            rc |= e->pack(w->ctx2att_w, H, A, H, e->p_ctx, st);
            rc |= e->pack_gates(w->att_lstm_w_ih, E + 2 * H, H, H, e->p_a_ih_h, st);
            rc |= e->pack_gates(w->att_lstm_w_ih + H, E + 2 * H, H, H, e->p_a_ih_fc, st);
            rc |= e->pack_gates(w->att_lstm_w_ih + 2 * H, E + 2 * H, H, E, e->p_a_ih_x, st);
            rc |= e->pack_gates(w->att_lstm_w_hh, H, H, H, e->p_a_hh, st);
            rc |= e->pack_gates(w->lang_lstm_w_ih, 2 * H, H, H, e->p_l_ih_a, st);
            rc |= e->pack_gates(w->lang_lstm_w_ih + H, 2 * H, H, H, e->p_l_ih_h, st);
            rc |= e->pack_gates(w->lang_lstm_w_hh, H, H, H, e->p_l_hh, st);
            rc |= e->pack(w->h2att_w, H, A, H, e->p_h2att, st);
        } else if (att2in2) {
            rc |= e->pack(w->att_embed_w, e->cfg.att_feat_size, H, e->cfg.att_feat_size, e->p_attw, st);
            rc |= e->pack(w->ctx2att_w, H, A, H, e->p_ctx, st);
            rc |= e->pack(w->h2att_w, H, A, H, e->p_h2att, st);
            rc |= e->pack(w->i2h_w, E, 5 * H, E, e->p_i2h, st);
            rc |= e->pack(w->h2h_w, H, 5 * H, H, e->p_h2h, st);
            rc |= e->pack(w->a2c_w, H, 2 * H, H, e->p_a2c, st);
        } else {
            rc |= e->pack(w->fc_embed_w, e->cfg.fc_feat_size, E, e->cfg.fc_feat_size, e->p_fc, st);
            rc |= e->pack(w->i2h_w, E, 5 * H, E, e->p_i2h, st);
            rc |= e->pack(w->h2h_w, H, 5 * H, H, e->p_h2h, st);
        }
        if (rc) return 1;
    }
    // per-token gate table: relu(embed)[V+1,E] * W_ih[:, 2H:2H+E]^T
    if (updown && build_gate_table(*e, w->embed, E, H, w->att_lstm_w_ih + 2 * H, E + 2 * H, e->p_a_ih_x, e->xgate, e->ld_xgate, st)) return 1;
    return e->finish_bind(st);
}

int capb200_engine_set_logit_layers(capb200_engine* e, int logit_layers) {
    CAPB_REQUIRE(e != nullptr, "null engine");
    return e->set_logit_layers(logit_layers, e->H);
}

int capb200_engine_bind_logit_head(capb200_engine* e, const float* const* w, const float* const* b, void* stream) {
    CAPB_REQUIRE(e != nullptr, "null engine");
    return e->bind_logit_head(w, b, static_cast<cudaStream_t>(stream));
}

int capb200_engine_bind_logit_head_grads(capb200_engine* e, float* const* gw, float* const* gb) {
    CAPB_REQUIRE(e != nullptr, "null engine");
    return e->bind_logit_head_grads(gw, gb);
}

int capb200_engine_set_logit_dropout(capb200_engine* e, float p) {
    CAPB_REQUIRE(e != nullptr, "null engine");
    return e->set_logit_dropout(p);
}

int capb200_decode_beam(capb200_engine* e, const float* fc, const float* att, const float* mask, int B, int R, const capb200_beam_opts* opts,
                        long long* seq, float* seq_logprobs, long long* done_seq, int* done_len, float* done_p, float* done_raw, void* stream) {
    return decode_beam(e, fc, att, mask, B, R, opts, seq, seq_logprobs, done_seq, done_len, done_p, done_raw, static_cast<cudaStream_t>(stream));
}

int capb200_decode_beam_form(int form, capb200_engine* e, const float* fc, const float* att, const float* mask, int B, int R,
                             const capb200_beam_opts* opts, long long* seq, float* seq_logprobs, long long* done_seq, int* done_len, float* done_p,
                             float* done_raw, void* stream) {
    return decode_beam(e, fc, att, mask, B, R, opts, seq, seq_logprobs, done_seq, done_len, done_p, done_raw, static_cast<cudaStream_t>(stream), form);
}

int capb200_decode_beam_diverse(capb200_engine* e, const float* fc, const float* att, const float* mask, int B, int R, const capb200_diverse_opts* opts,
                                long long* seq, float* seq_logprobs, long long* done_seq, int* done_len, float* done_p, float* done_raw, void* stream) {
    return decode_beam_diverse(e, fc, att, mask, B, R, opts, seq, seq_logprobs, done_seq, done_len, done_p, done_raw, static_cast<cudaStream_t>(stream));
}

int capb200_beam_record_logprobs(capb200_engine* e, int image, int rank, float* dst, void* stream) {
    return decode_record_logprobs(e, image, rank, dst, static_cast<cudaStream_t>(stream));
}

int capb200_decode_sample(capb200_engine* e, const float* fc, const float* att, const float* mask, int B, int R, const capb200_sample_opts* opts,
                          const long long* tokens_in, long ld_tok, long long* seq, float* seq_logprobs, float* picked, void* stream) {
    return decode_sample(e, fc, att, mask, B, R, opts, tokens_in, ld_tok, seq, seq_logprobs, picked, static_cast<cudaStream_t>(stream));
}

// ---------------------------------------------------------------------------------------------------------------------
// operator-level entry points
// ---------------------------------------------------------------------------------------------------------------------
int capb200_linear(const float* x, long ldx, const float* w, long ldw, const float* b, float* y, long ldy, int M, int N, int K, int relu, int mode,
                   void* stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CAPB_REQUIRE(x && w && y && M > 0 && N > 0 && K > 0, "bad argument");
    GemmProblem g;
    g.M = M; g.N = N; g.nseg = 1;
    g.seg[0].A = x; g.seg[0].lda = ldx; g.seg[0].W = w; g.seg[0].ldw = ldw; g.seg[0].K = K;
    g.epi.bias = b; g.epi.relu = relu; g.epi.C = y; g.epi.ldc = ldy;
    if (mode == CAPB200_MODE_SIMT_FP32) return gemm_simt_launch(g, st);
    if (mode == CAPB200_MODE_SKINNY_TF32X3 || mode == CAPB200_MODE_SKINNY_FP32) {
        // the training step's split-K GEMM (no relu epilogue); scratch for the partial sums is allocated per call here
        CAPB_REQUIRE(!relu, "the skinny GEMM has no relu epilogue");
        const size_t cap = (size_t)4 << 20;
        float* part = nullptr;
        CAPB_CHECK_CUDA(cudaMallocAsync(&part, cap * sizeof(float), st));
        const int tb = 1;
        const int rc = gemm_skinny_launch(M, N, 1, &x, &ldx, &w, &ldw, &K, &tb, y, ldy, b, nullptr, 0, 1, 0, part, cap, mode == CAPB200_MODE_SKINNY_TF32X3, st);
        cudaFreeAsync(part, st);
        return rc;
    }
    if (mode == CAPB200_MODE_TF32X3_TC || mode == CAPB200_MODE_TF32X3_TC_DGRAD || mode == CAPB200_MODE_TF32X3_TC_WGRAD) {
        // the training steps' wgmma tf32 kernel (gemm_tf32.cu) through the same helper the engines use:
        //   TF32X3_TC        y[M,N]  = x[M,K] w[N,K]^T + b                         (forward)
        //   TF32X3_TC_DGRAD  y[M,N]  = x[M,K] w'[K,N]       with w' passed as `w`  (input gradient: W stored [out = K, in = N], cached transpose)
        //   TF32X3_TC_WGRAD  y[M,N]  = x'[K,M]^T w'[K,N]    with x', w' row-major   (weight gradient: dY = x', X = w', transposed per call)
        CAPB_REQUIRE(!relu, "the tf32 GEMM has no relu epilogue");
        Tf32Context* ctx = tf32_context_create();
        Skinny sk{nullptr, 0, 1, st};
        sk.ctx = ctx;
        int rc;
        if (mode == CAPB200_MODE_TF32X3_TC) rc = sk.lin(x, ldx, w, ldw, b, y, ldy, M, N, K, 0);
        else if (mode == CAPB200_MODE_TF32X3_TC_DGRAD) rc = sk.dgrad(M, N, K, x, ldx, w, ldw, y, ldy, 0);
        else rc = sk.wgrad(M, N, K, x, ldx, w, ldw, y, ldy, 0);
        if (tf32_context_launches(ctx) == 0 && !rc) { set_error("capb200_linear: the operands are not TMA-compatible, the wgmma tf32 kernel did not run"); rc = 1; }
        cudaStreamSynchronize(st);
        tf32_context_destroy(ctx);
        return rc;
    }
    CAPB_REQUIRE(mode == CAPB200_MODE_TC_F16X3 || mode == CAPB200_MODE_TC_F16X1, "unknown mode");
    const long ldh = round_up(K, 64);
    __half* scratch = nullptr;
    const size_t elems = (size_t)(M + N) * ldh * 2;
    CAPB_CHECK_CUDA(cudaMallocAsync(&scratch, elems * sizeof(__half), st));
    __half* xh = scratch; __half* xl = xh + (size_t)M * ldh;
    __half* wh = xl + (size_t)M * ldh; __half* wl = wh + (size_t)N * ldh;
    int rc = split_planes_launch(x, ldx, M, K, xh, xl, ldh, st) | split_planes_launch(w, ldw, N, K, wh, wl, ldh, st);
    g.seg[0].A_hi = xh; g.seg[0].A_lo = xl; g.seg[0].lda_h = ldh;
    g.seg[0].W_hi = wh; g.seg[0].W_lo = wl; g.seg[0].ldw_h = ldh;
    GemmTcPlan* plan = rc ? nullptr : gemm_tc_plan_create(g, mode == CAPB200_MODE_TC_F16X3 ? 3 : 1);
    if (plan == nullptr) rc = 1;
    if (!rc) rc = gemm_tc_plan_launch(plan, nullptr, 0, st);
    if (plan) gemm_tc_plan_destroy(plan);
    cudaFreeAsync(scratch, st);
    return rc;
}

int capb200_bench_linear(const float* x, const float* w, const float* b, float* y, int M, int N, int K, int mode, int iters, float* ms_per_launch,
                         void* stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CAPB_REQUIRE(x && w && y && ms_per_launch && M > 0 && N > 0 && K > 0 && iters > 0, "bad argument");
    if (mode == CAPB200_MODE_TF32X3_TC || mode == CAPB200_MODE_SKINNY_TF32X3) {
        // the training GEMMs: wgmma tf32 kernel (gemm_tf32.cu) or the mma.sync split-K kernel it replaced, timed back to back
        Tf32Context* ctx = mode == CAPB200_MODE_TF32X3_TC ? tf32_context_create() : nullptr;
        float* scratch = nullptr;
        const size_t cap = (size_t)4 << 20;
        CAPB_CHECK_CUDA(cudaMalloc(&scratch, cap * sizeof(float)));
        Skinny sk{scratch, cap, 1, st};
        sk.ctx = ctx;
        cudaEvent_t e0, e1;
        cudaEventCreate(&e0);
        cudaEventCreate(&e1);
        int rc = 0;
        for (int i = 0; i < 3 + iters && !rc; ++i) {
            if (i == 3) cudaEventRecord(e0, st);
            rc = sk.lin(x, K, w, K, b, y, N, M, N, K, 0);
        }
        cudaEventRecord(e1, st);
        if (cudaStreamSynchronize(st) != cudaSuccess) { set_error(std::string("bench_linear: ") + cudaGetErrorString(cudaGetLastError())); rc = 1; }
        float ms = 0.f;
        if (!rc) { cudaEventElapsedTime(&ms, e0, e1); *ms_per_launch = ms / iters; }
        cudaEventDestroy(e0);
        cudaEventDestroy(e1);
        cudaFree(scratch);
        tf32_context_destroy(ctx);
        return rc;
    }
    GemmProblem g;
    g.M = M; g.N = N; g.nseg = 1;
    g.seg[0].A = x; g.seg[0].lda = K; g.seg[0].W = w; g.seg[0].ldw = K; g.seg[0].K = K;
    g.epi.bias = b; g.epi.C = y; g.epi.ldc = N;
    const long ldh = round_up(K, 64);
    __half* scratch = nullptr;
    GemmTcPlan* plan = nullptr;
    int rc = 0;
    if (mode != CAPB200_MODE_SIMT_FP32) {
        CAPB_CHECK_CUDA(cudaMalloc(&scratch, (size_t)(M + N) * ldh * 2 * sizeof(__half)));
        __half* xh = scratch; __half* xl = xh + (size_t)M * ldh;
        __half* wh = xl + (size_t)M * ldh; __half* wl = wh + (size_t)N * ldh;
        rc = split_planes_launch(x, K, M, K, xh, xl, ldh, st) | split_planes_launch(w, K, N, K, wh, wl, ldh, st);
        g.seg[0].A_hi = xh; g.seg[0].A_lo = xl; g.seg[0].lda_h = ldh;
        g.seg[0].W_hi = wh; g.seg[0].W_lo = wl; g.seg[0].ldw_h = ldh;
        plan = rc ? nullptr : gemm_tc_plan_create(g, mode == CAPB200_MODE_TC_F16X3 ? 3 : 1);
        if (plan == nullptr) rc = 1;
    }
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    for (int i = 0; i < 3 + iters && !rc; ++i) {
        if (i == 3) cudaEventRecord(e0, st);
        rc = plan ? gemm_tc_plan_launch(plan, nullptr, 0, st) : gemm_simt_launch(g, st);
    }
    cudaEventRecord(e1, st);
    if (cudaStreamSynchronize(st) != cudaSuccess) { set_error(std::string("bench_linear: ") + cudaGetErrorString(cudaGetLastError())); rc = 1; }
    float ms = 0.f;
    if (!rc) { cudaEventElapsedTime(&ms, e0, e1); *ms_per_launch = ms / iters; }
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    if (plan) gemm_tc_plan_destroy(plan);
    if (scratch) cudaFree(scratch);
    return rc;
}

int capb200_decode_gemm(const float* x, const float* w, int M, int N, int K, int mode, const capb200_gemm_epilogue* epi, unsigned long long* trace_host,
                        int n_slots, void* stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CAPB_REQUIRE(x && w && epi && M > 0 && N > 0 && K > 0, "bad argument");
    CAPB_REQUIRE(mode == CAPB200_MODE_TC_F16X3 || mode == CAPB200_MODE_TC_F16X1, "the decode GEMM runs in the tc_f16x3 / tc_f16x1 modes");
    CAPB_REQUIRE(trace_host == nullptr || (n_slots >= 296 * 16 && mode == CAPB200_MODE_TC_F16X3), "the trace needs 296 x 16 slots and tc_f16x3");
    GemmProblem g;
    g.M = M; g.N = N; g.nseg = 1;
    g.seg[0].K = K;
    GemmEpilogue& e = g.epi;
    e.bias = epi->bias; e.row_bias = epi->row_bias; e.ld_row_bias = epi->ld_row_bias; e.rows_per_group = epi->rows_per_group;
    e.residual = epi->residual; e.ld_res = epi->ld_res; e.relu = epi->relu;
    e.C = epi->C; e.ldc = epi->ldc;
    e.C_hi = reinterpret_cast<__half*>(epi->C_hi); e.C_lo = reinterpret_cast<__half*>(epi->C_lo); e.ldcs = epi->ldcs;
    e.lstm = epi->lstm; e.H = epi->H;
    e.c_prev = epi->c_prev; e.ld_cprev = epi->ld_cprev; e.src_row = epi->src_row;
    e.c_out = epi->c_out; e.ld_cout = epi->ld_cout;
    e.gather_bias = epi->gather_bias; e.ld_gb = epi->ld_gb; e.gather_idx = epi->gather_idx;
    e.h_f = epi->h_f; e.h_hi = reinterpret_cast<__half*>(epi->h_hi); e.h_lo = reinterpret_cast<__half*>(epi->h_lo); e.ld_h = epi->ld_h;
    CAPB_REQUIRE(e.C_hi == nullptr || e.C_lo != nullptr, "C_hi needs C_lo");
    CAPB_REQUIRE(e.h_hi == nullptr || e.h_lo != nullptr, "h_hi needs h_lo");
    CAPB_REQUIRE(e.row_bias == nullptr || e.rows_per_group >= 1, "rows_per_group must be >= 1");
    CAPB_REQUIRE(e.gather_bias == nullptr || e.gather_idx != nullptr, "gather_bias needs gather_idx");
    const long ldh = round_up(K, 64);
    __half* scratch = nullptr;
    unsigned long long* trace = nullptr;
    CAPB_CHECK_CUDA(cudaMalloc(&scratch, (size_t)(M + N) * ldh * 2 * sizeof(__half)));
    if (trace_host != nullptr) {
        CAPB_CHECK_CUDA(cudaMalloc(&trace, sizeof(unsigned long long) * 296 * 16));
        CAPB_CHECK_CUDA(cudaMemsetAsync(trace, 0, sizeof(unsigned long long) * 296 * 16, st));
    }
    __half* xh = scratch; __half* xl = xh + (size_t)M * ldh;
    __half* wh = xl + (size_t)M * ldh; __half* wl = wh + (size_t)N * ldh;
    int rc = split_planes_launch(x, K, M, K, xh, xl, ldh, st) | split_planes_launch(w, K, N, K, wh, wl, ldh, st);
    g.seg[0].A_hi = xh; g.seg[0].A_lo = xl; g.seg[0].lda_h = ldh;
    g.seg[0].W_hi = wh; g.seg[0].W_lo = wl; g.seg[0].ldw_h = ldh;
    GemmTcPlan* plan = rc ? nullptr : gemm_tc_plan_create(g, mode == CAPB200_MODE_TC_F16X3 ? 3 : 1);
    if (plan == nullptr) rc = 1;
    // traced: three warm launches first, so the stamps show the steady state (outputs must not overlap inputs)
    for (int i = 0; i < (trace ? 3 : 1) && !rc; ++i) rc = gemm_tc_plan_launch(plan, nullptr, 0, st);
    if (!rc && trace) {
        GemmEpilogue ep = g.epi;
        ep.trace = trace;
        rc = gemm_tc_plan_launch(plan, &ep, 0, st);
    }
    if (cudaStreamSynchronize(st) != cudaSuccess) { set_error(std::string("decode_gemm: ") + cudaGetErrorString(cudaGetLastError())); rc = 1; }
    if (!rc && trace) CAPB_CHECK_CUDA(cudaMemcpy(trace_host, trace, sizeof(unsigned long long) * 296 * 16, cudaMemcpyDeviceToHost));
    if (plan) gemm_tc_plan_destroy(plan);
    cudaFree(scratch);
    if (trace) cudaFree(trace);
    return rc;
}

int capb200_gemm_tile_n(int M, int N) { return gemm_tc_tile_n(M, N); }

int capb200_gemm_tile_m(int M, int N) { return gemm_tc_tile_m(M, N, gemm_tc_tile_n(M, N)); }

int capb200_lstm_cell(const float* x, int Kx, const float* h, const float* c, const float* w_ih, const float* w_hh, const float* b_ih,
                      const float* b_hh, float* h_out, float* c_out, int M, int H, int mode, void* stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CAPB_REQUIRE(x && h && c && w_ih && w_hh && b_ih && b_hh && h_out && c_out, "null argument");
    float* gates = nullptr;
    CAPB_CHECK_CUDA(cudaMallocAsync(&gates, sizeof(float) * ((size_t)M * 4 * H + 4 * H), st));
    float* bsum = gates + (size_t)M * 4 * H;
    add_vec_kernel<<<cdiv(4 * H, 256), 256, 0, st>>>(b_ih, b_hh, bsum, 4 * H);
    int rc = capb200_linear(x, Kx, w_ih, Kx, bsum, gates, 4 * H, M, 4 * H, Kx, 0, mode, stream);
    float* g2 = nullptr;
    if (!rc) {
        // second contraction accumulated through a temporary: gates += h * w_hh^T
        CAPB_CHECK_CUDA(cudaMallocAsync(&g2, sizeof(float) * (size_t)M * 4 * H, st));
        rc = capb200_linear(h, H, w_hh, H, nullptr, g2, 4 * H, M, 4 * H, H, 0, mode, stream);
        if (!rc) add_vec_kernel<<<cdiv(M * 4 * H, 256), 256, 0, st>>>(gates, g2, gates, M * 4 * H);
    }
    if (!rc) {
        ActView ho; ho.f = h_out; ho.ld = H;
        rc = lstm_pointwise_launch(M, H, gates, 4 * H, nullptr, c, H, c_out, H, ho, nullptr, 0, nullptr, st);
    }
    if (g2) cudaFreeAsync(g2, st);
    cudaFreeAsync(gates, st);
    return rc;
}

int capb200_additive_attention(const float* att_h, const float* p_att, const float* att, const float* mask, const float* alpha_w,
                               const float* alpha_b, float* out, int n_images, int rows_per_image, int R, int A, int H, void* stream) {
    CAPB_REQUIRE(att_h && p_att && att && alpha_w && alpha_b && out, "null argument");
    ActView o; o.f = out; o.ld = H;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    float* scratch = nullptr;
    CAPB_CHECK_CUDA(cudaMallocAsync(&scratch, sizeof(float) * (size_t)n_images * rows_per_image * R, st));
    const int rc = additive_attention_launch(n_images, rows_per_image, R, A, H, att_h, A, p_att, A, att, H, mask, R, alpha_w, alpha_b, scratch, o, st);
    cudaFreeAsync(scratch, st);
    return rc;
}

int capb200_log_softmax_topk(float* logits, long ld, int rows, int V1, int twice, int k, float* top_val, int* top_idx, void* stream) {
    CAPB_REQUIRE(logits != nullptr && rows > 0 && V1 > 0, "bad argument");
    VocabStepArgs va;
    va.rows = rows; va.V1 = V1; va.logits = logits; va.ld = ld; va.twice = twice; va.topk = k; va.top_val = top_val; va.top_idx = top_idx;
    return vocab_step_launch(va, static_cast<cudaStream_t>(stream));
}

int capb200_vocab_stats_topk(const float* logits, long ld, int rows, int V1, int twice, int k, float* stats, float* top_val, int* top_idx, void* stream) {
    CAPB_REQUIRE(logits != nullptr && stats != nullptr && top_val != nullptr && top_idx != nullptr, "null argument");
    CAPB_REQUIRE(rows > 0 && V1 > 0 && ld >= V1 && k > 0, "bad argument");
    CAPB_REQUIRE((reinterpret_cast<uintptr_t>(stats) & 7) == 0, "stats must be 8-byte aligned");
    VocabStepArgs va;
    va.rows = rows; va.V1 = V1; va.logits = const_cast<float*>(logits); va.ld = ld; va.twice = twice;      // stats mode only reads the rows
    va.topk = k; va.top_val = top_val; va.top_idx = top_idx;
    va.stats = reinterpret_cast<float2*>(stats);
    return vocab_step_launch(va, static_cast<cudaStream_t>(stream));
}

int capb200_vocab_select(float* logits, long ld, int rows, int V1, int select, float top, float temperature, unsigned long long seed,
                         unsigned long long step, int* unfinished, int first_step, int* tokens_out, float* picked_lp, void* stream) {
    CAPB_REQUIRE(logits != nullptr && tokens_out != nullptr && picked_lp != nullptr, "null argument");
    CAPB_REQUIRE(rows > 0 && V1 > 0 && ld >= V1, "bad argument");
    CAPB_REQUIRE(select == 1 || select == 2 || select == 4 || select == 5, "select must be 1 (greedy), 2 (multinomial), 4 (top-k) or 5 (nucleus)");
    CAPB_REQUIRE(temperature > 0.f, "temperature must be positive");
    CAPB_REQUIRE(select != 4 || top >= 1.f, "top-k sampling needs k >= 1");
    CAPB_REQUIRE(select != 5 || (top > 0.f && top <= 1.f), "nucleus sampling needs 0 < p <= 1");
    VocabStepArgs va;
    va.rows = rows; va.V1 = V1; va.logits = logits; va.ld = ld;
    va.select = select; va.top = top; va.temperature = temperature; va.seed = seed; va.step = step;
    va.unfinished = unfinished; va.first_step = first_step; va.tokens_out = tokens_out; va.picked_lp = picked_lp;
    return vocab_step_launch(va, static_cast<cudaStream_t>(stream));
}

}  // extern "C"

// =====================================================================================================================
// Training steps (UpDown, Att2in2, NewFC) on the scaffold of train_common.cuh
// =====================================================================================================================
namespace {

// UpDown's tape: the forward [T][N][.] except out [N][T][H], the prologue, and the gradients carried through time
struct Tape : StepTape {
    int* tok;
    float *xt, *g1, *h0, *c0, *atth, *alpha, *attres, *g2, *h1, *c1, *out;
    float *fc_e, *att_e, *p_att, *g_fc;
    float *dOUT, *DG1, *DG2, *DATTH, *dh0, *dc0, *dh1, *dc1, *tmpH, *dX2, *dxt, *d_att_e, *d_p_att, *S, *d_fc_e, *dpre_att, *dpre_fc, *dalpha;
    float* s_att_score;
};

void layout_tape(Tape& tp, Arena& a, int B, int R, int N, int T, int E, int H, int A, int V1) {
    const long TN = (long)T * N, BR = (long)B * R;
    tp.layout(a, B, N, TN, V1, (long)B * T * V1);
    tp.tok = a.take<int>(TN);
    tp.xt = a.take<float>(TN * E); tp.g1 = a.take<float>(TN * 4 * H); tp.h0 = a.take<float>(TN * H); tp.c0 = a.take<float>(TN * H);
    tp.atth = a.take<float>(TN * A); tp.alpha = a.take<float>(TN * R); tp.attres = a.take<float>(TN * H);
    tp.g2 = a.take<float>(TN * 4 * H); tp.h1 = a.take<float>(TN * H); tp.c1 = a.take<float>(TN * H); tp.out = a.take<float>(TN * H);
    tp.fc_e = a.take<float>((long)B * H); tp.att_e = a.take<float>(BR * H); tp.p_att = a.take<float>(BR * A); tp.g_fc = a.take<float>((long)B * 4 * H);
    tp.dOUT = a.take<float>(TN * H); tp.DG1 = a.take<float>(TN * 4 * H); tp.DG2 = a.take<float>(TN * 4 * H);
    tp.DATTH = a.take<float>(TN * A);
    tp.dh0 = a.take<float>((long)N * H); tp.dc0 = a.take<float>((long)N * H); tp.dh1 = a.take<float>((long)N * H); tp.dc1 = a.take<float>((long)N * H);
    tp.tmpH = a.take<float>((long)N * H); tp.dX2 = a.take<float>((long)N * 2 * H); tp.dxt = a.take<float>((long)N * E);
    tp.d_att_e = a.take<float>(BR * H); tp.d_p_att = a.take<float>(BR * A); tp.S = a.take<float>((long)B * 4 * H); tp.d_fc_e = a.take<float>((long)B * H);
    tp.dpre_att = a.take<float>(BR * H); tp.dpre_fc = a.take<float>((long)B * H);
    tp.dalpha = a.take<float>((long)N * R);
    tp.s_att_score = a.take<float>((long)N * R);
}

// The tape of the maxout-cell families (Att2in2, NewFC).  sums / DS hold the maxout sums (i, f, o, a, b) and their gradient [T][N][5H];
// h / c hold T+1 slots (slot 0 = the initial state, slot t+1 = step t), so step t -- and the batched weight gradients of h2h and h2att --
// read the previous state from slot t.
struct MaxoutTape : StepTape {
    int* tok;
    float *xt, *sums, *h, *c, *out, *dOUT, *DS, *dh, *dc, *dxt;
    // Att2in2's attention on the previous h
    float *atth, *alpha, *attres, *att_e, *p_att, *DATTH, *d_attres, *d_att_e, *d_p_att, *dpre_att, *dalpha, *s_att_score;
    // NewFC's image step on B rows: fc_e [B, E] = fc_embed(fc), its maxout sums and state and their gradients; img_row = the image of each row
    float *fc_e, *d_fc_e, *im_sums, *im_ds, *im_h, *im_c, *im_dh, *im_dc;
    int* img_row;
};

void layout_maxout_tape(MaxoutTape& tp, Arena& a, int B, int R, int N, int T, int E, int H, int A, int V1) {
    const long TN = (long)T * N, BR = (long)B * R, NH = (long)N * H;
    tp = MaxoutTape{};
    tp.layout(a, B, N, TN, V1, (long)B * T * V1);
    tp.tok = a.take<int>(TN);
    tp.xt = a.take<float>(TN * E); tp.sums = a.take<float>(TN * 5 * H); tp.h = a.take<float>(TN * H + NH); tp.c = a.take<float>(TN * H + NH);
    tp.out = a.take<float>(TN * H); tp.dOUT = a.take<float>(TN * H); tp.DS = a.take<float>(TN * 5 * H);
    tp.dh = a.take<float>(NH); tp.dc = a.take<float>(NH); tp.dxt = a.take<float>((long)N * E);
    tp.atth = a.take<float>(TN * A); tp.alpha = a.take<float>(TN * R); tp.attres = a.take<float>(TN * H);
    tp.att_e = a.take<float>(BR * H); tp.p_att = a.take<float>(BR * A); tp.DATTH = a.take<float>(TN * A); tp.d_attres = a.take<float>(NH);
    tp.d_att_e = a.take<float>(BR * H); tp.d_p_att = a.take<float>(BR * A); tp.dpre_att = a.take<float>(BR * H);
    tp.dalpha = a.take<float>((long)N * R); tp.s_att_score = a.take<float>((long)N * R);
}

// NewFC: the maxout tape without the attention, plus the image step
void layout_newfc_tape(MaxoutTape& tp, Arena& a, int B, int N, int T, int E, int H, int V1) {
    layout_maxout_tape(tp, a, B, 0, N, T, E, H, 0, V1);
    tp.fc_e = a.take<float>((long)B * E); tp.d_fc_e = a.take<float>((long)B * E);
    tp.im_sums = a.take<float>((long)B * 5 * H); tp.im_ds = a.take<float>((long)B * 5 * H);
    tp.im_h = a.take<float>((long)B * H); tp.im_c = a.take<float>((long)B * H);
    tp.im_dh = a.take<float>((long)B * H); tp.im_dc = a.take<float>((long)B * H);
    tp.img_row = a.take<int>(N);
}

}  // namespace

extern "C" int capb200_dropout_mask(float* mask, long n, unsigned long long seed, int site, int step, float p, void* stream) {
    CAPB_REQUIRE(mask != nullptr && n > 0, "bad argument");
    if (dropout_salt_set_all(0ull, static_cast<cudaStream_t>(stream))) return 1;      // a graph replay of an SCST step may have left a salt behind
    return dropout_mask_launch(mask, n, seed, (unsigned)site, (unsigned)step, p, static_cast<cudaStream_t>(stream));
}

namespace {

// (1) of an SCST step with the eval-mode baseline: fork it and enqueue it right away on this engine's decode path (NewFC: att = null, R = 0).
int start_baseline(capb200_engine* e, const float* fc, const float* att, int B, int R, const TrainArgs& ta, const StepTape& tp, StepBaseline& gb,
                          cudaStream_t st) {
    if (gb.fork(ta, &e->side, &e->ev_fork, &e->ev_join, st)) return 1;
    return gb.enqueue(B, ta.T, e->V1, ta.greedy_seq, tp.glp, [&](const capb200_sample_opts* so, const long long* tok, long long* seq, float* lp, void* s) {
        return capb200_decode_sample(e, fc, att, ta.mask, B, R, so, tok, tok ? ta.T : 0, seq, lp, nullptr, s);
    });
}

// The attention prologue UpDown and Att2in2 share, on the tape: att_embed (ReLU, dropout site 1, padded regions zeroed) and ctx2att.
template <class Tp>
int att_prologue_forward(capb200_engine* e, const Skinny& sk, Tp& tp, const float* att, int B, int R, const float* mask, unsigned long long seed, float p,
                         cudaStream_t st) {
    const int H = e->H, A = e->A, Fa = e->cfg.att_feat_size, BR = B * R;
    const capb200_weights& w = e->w;
    if (sk.lin(att, Fa, w.att_embed_w, Fa, w.att_embed_b, tp.att_e, H, BR, H, Fa, 0)) return 1;
    if (relu_copy_launch(tp.att_e, (long)BR * H, f32_view(tp.att_e, H), st)) return 1;
    if (dropout_apply_launch(tp.att_e, BR, H, H, seed, 1, 0, p, st)) return 1;
    if (mask != nullptr) {      // pack_wrapper: the embedding of a padded region is exactly zero (AttModel.py:44-49); relu'(0) = 0 keeps its gradient zero
        if (mask_rows_launch(f32_view(tp.att_e, H), B, R, H, mask, R, st)) return 1;
        e->launches++;
    }
    if (sk.lin(tp.att_e, H, w.ctx2att_w, H, w.ctx2att_b, tp.p_att, A, BR, A, H, 0)) return 1;
    e->launches += 4;
    return 0;
}

// Its backward: d att_e += d p_att * ctx2att, then the ctx2att and att_embed gradients (keep_scale = 1 / (1 - p)).
template <class Tp, class Grads>
int att_prologue_backward(capb200_engine* e, const Skinny& sk, const Tp& tp, const float* att, int B, int R, float keep_scale, const Grads& G, cudaStream_t st) {
    const int H = e->H, A = e->A, Fa = e->cfg.att_feat_size, BR = B * R;
    int rc = 0;
    rc |= sk.dgrad(BR, H, A, tp.d_p_att, A, e->w.ctx2att_w, H, tp.d_att_e, H, 1);
    rc |= sk.wgrad(A, H, BR, tp.d_p_att, A, tp.att_e, H, G.ctx2att_w, H, 0);
    rc |= colsum_launch(BR, A, tp.d_p_att, A, G.ctx2att_b, 0, st);
    rc |= relu_dropout_backward_launch((long)BR * H, tp.att_e, tp.d_att_e, tp.dpre_att, keep_scale, st);
    rc |= sk.wgrad(H, Fa, BR, tp.dpre_att, H, att, Fa, G.att_embed_w, Fa, 0);
    rc |= colsum_launch(BR, H, tp.dpre_att, H, G.att_embed_b, 0, st);
    e->launches += 6;
    return rc;
}

int updown_train_step(capb200_engine* e, const float* fc, const float* att, int B, int R, const TrainArgs& ta, const capb200_updown_grads* grads,
                      cudaStream_t st) {
    const int n = ta.n, N = B * n, T = ta.T, E = e->E, H = e->H, A = e->A, V1 = e->V1;
    const int Ff = e->cfg.fc_feat_size;
    const float p = ta.p;
    const float keep_scale = 1.0f / (1.0f - p);
    const unsigned long long seed = ta.seed;
    const capb200_weights& w = e->w;
    const long ld_lp = (long)ta.Tl * V1;

    // ---- (1) greedy baseline, eval mode (no dropout): the regular decode path
    Tape tp;
    if (carve_tape(&e->tape, &e->tape_bytes, tp, st, [&](Tape& t, Arena& a) { layout_tape(t, a, B, R, N, T, E, H, A, V1); })) return 1;
    if (head_train_tape(e, (long)T * N, st)) return 1;
    if (ensure_workspace(e, B, N, R, 1, st)) return 1;        // decode workspace sized before anything is in flight
    StepBaseline gb;
    if (start_baseline(e, fc, att, B, R, ta, tp, gb, st)) return 1;
    const Skinny sk = step_gemms(&e->tf32, e->tc, tp, st);
    const long tf32_l0 = tf32_context_launches(e->tf32);

    // ---- (2) train-mode prologue: fc_embed / att_embed with dropout, ctx2att, per-image gate term
    nvtxRangePushA("capb200 train step: forward on the tape");
    const long BR = (long)B * R;
    if (sk.lin(fc, Ff, w.fc_embed_w, Ff, w.fc_embed_b, tp.fc_e, H, B, H, Ff, 0)) return 1;
    if (relu_copy_launch(tp.fc_e, (long)B * H, f32_view(tp.fc_e, H), st)) return 1;
    if (dropout_apply_launch(tp.fc_e, B, H, H, seed, 0, 0, p, st)) return 1;
    if (att_prologue_forward(e, sk, tp, att, B, R, ta.mask, seed, p, st)) return 1;
    if (sk.lin(tp.fc_e, H, w.att_lstm_w_ih + H, E + 2 * H, e->bsum_att, tp.g_fc, 4 * H, B, 4 * H, H, 0)) return 1;
    e->launches += 4;

    // ---- (3) T sampling steps with the tape
    const long NH = (long)N * H;
    CAPB_CHECK_CUDA(cudaMemsetAsync(tp.s_tokens, 0, sizeof(int) * N, st));
    for (int t = 0; t < T; ++t) {
        int* tok = tp.tok + (long)t * N;
        if (feed_tokens(ta, tp, N, V1, t, tok, st)) return 1;
        float* xt = tp.xt + (long)t * N * E;
        float* g1 = tp.g1 + (long)t * N * 4 * H;
        float* g2 = tp.g2 + (long)t * N * 4 * H;
        const float* h0p = t ? tp.h0 + (long)(t - 1) * NH : nullptr;
        const float* h1p = t ? tp.h1 + (long)(t - 1) * NH : nullptr;
        const float* c0p = t ? tp.c0 + (long)(t - 1) * NH : nullptr;
        const float* c1p = t ? tp.c1 + (long)(t - 1) * NH : nullptr;
        float *h0 = tp.h0 + (long)t * NH, *c0 = tp.c0 + (long)t * NH, *h1 = tp.h1 + (long)t * NH, *c1 = tp.c1 + (long)t * NH;
        if (embed_relu_dropout_launch(N, E, tok, w.embed, xt, seed, (unsigned)t, p, st)) return 1;
        // gates1 = g_fc[img] + xt W_x^T (+ h_lang_prev W_h^T + h_att_prev W_hh^T)
        {
            GemmProblem g; g.M = N; g.N = 4 * H; g.nseg = 1;
            g.seg[0].A = xt; g.seg[0].lda = E; g.seg[0].W = w.att_lstm_w_ih + 2 * H; g.seg[0].ldw = E + 2 * H; g.seg[0].K = E;
            if (t) {
                g.seg[1].A = h1p; g.seg[1].lda = H; g.seg[1].W = w.att_lstm_w_ih; g.seg[1].ldw = E + 2 * H; g.seg[1].K = H;
                g.seg[2].A = h0p; g.seg[2].lda = H; g.seg[2].W = w.att_lstm_w_hh; g.seg[2].ldw = H; g.seg[2].K = H;
                g.nseg = 3;
            }
            g.epi.row_bias = tp.g_fc; g.epi.ld_row_bias = 4 * H; g.epi.rows_per_group = n;
            g.epi.C = g1; g.epi.ldc = 4 * H;
            if (sk.gates(g)) return 1;
        }
        if (lstm_pointwise_launch(N, H, g1, 4 * H, nullptr, c0p, H, c0, H, f32_view(h0, H), nullptr, 0, nullptr, st)) return 1;
        float* atth = tp.atth + (long)t * N * A;
        if (sk.lin(h0, H, w.h2att_w, H, w.h2att_b, atth, A, N, A, H, 0)) return 1;
        float* attres = tp.attres + (long)t * NH;
        if (additive_attention_launch(B, n, R, A, H, atth, A, tp.p_att, A, tp.att_e, H, ta.mask, R, w.alpha_w, w.alpha_b, tp.s_att_score,
                                      f32_view(attres, H), st, tp.alpha + (long)t * N * R)) return 1;
        {
            GemmProblem g; g.M = N; g.N = 4 * H; g.nseg = 2;
            g.seg[0].A = attres; g.seg[0].lda = H; g.seg[0].W = w.lang_lstm_w_ih; g.seg[0].ldw = 2 * H; g.seg[0].K = H;
            g.seg[1].A = h0; g.seg[1].lda = H; g.seg[1].W = w.lang_lstm_w_ih + H; g.seg[1].ldw = 2 * H; g.seg[1].K = H;
            if (t) { g.seg[2].A = h1p; g.seg[2].lda = H; g.seg[2].W = w.lang_lstm_w_hh; g.seg[2].ldw = H; g.seg[2].K = H; g.nseg = 3; }
            g.epi.bias = e->bsum_lang;
            g.epi.C = g2; g.epi.ldc = 4 * H;
            if (sk.gates(g)) return 1;
        }
        if (lstm_pointwise_launch(N, H, g2, 4 * H, nullptr, c1p, H, c1, H, f32_view(h1, H), nullptr, 0, nullptr, st)) return 1;
        // core output = dropout(h_lang), stored in (n, t) order for the batched logit backward
        float* out = tp.out + (long)t * H;
        if (dropout_copy_launch(h1, H, out, (long)T * H, N, H, seed, 3, (unsigned)t, p, st)) return 1;
        const float* lin_in;
        long ld_in;
        if (head_train_forward(e, sk, out, (long)T * H, N, T, t, seed, &lin_in, &ld_in, st)) return 1;
        if (sk.lin(lin_in, ld_in, w.logit_w, H, w.logit_b, ta.logprobs + (long)t * V1, ld_lp, N, V1, H, 0)) return 1;
        if (train_vocab_step(ta, tp, N, V1, t, st)) return 1;
        e->launches += 12;
    }

    // ---- (4) reward and loss, (5) the logit layer's backward
    nvtxRangePop();
    if (ta.forward_only) return 0;
    CAPB_NVTX("capb200 train step: reward, loss, backward through time, weight gradients");
    const long TN = (long)T * N;
    const capb200_updown_grads& G = *grads;
    if (loss_and_logit_backward(e, ta, tp, gb, sk, B, N, V1, H, w.logit_w, tp.out, tp.dOUT, G.logit_w, G.logit_b, e->grad_events[0], st)) return 1;
    CAPB_CHECK_CUDA(cudaMemsetAsync(tp.dh0, 0, sizeof(float) * NH, st));
    CAPB_CHECK_CUDA(cudaMemsetAsync(tp.dc0, 0, sizeof(float) * NH, st));
    CAPB_CHECK_CUDA(cudaMemsetAsync(tp.dh1, 0, sizeof(float) * NH, st));
    CAPB_CHECK_CUDA(cudaMemsetAsync(tp.dc1, 0, sizeof(float) * NH, st));
    CAPB_CHECK_CUDA(cudaMemsetAsync(tp.d_att_e, 0, sizeof(float) * BR * H, st));
    CAPB_CHECK_CUDA(cudaMemsetAsync(tp.d_p_att, 0, sizeof(float) * BR * A, st));
    CAPB_CHECK_CUDA(cudaMemsetAsync(G.alpha_w, 0, sizeof(float) * A, st));
    CAPB_CHECK_CUDA(cudaMemsetAsync(G.alpha_b, 0, sizeof(float), st));
    CAPB_CHECK_CUDA(cudaMemsetAsync(G.embed, 0, sizeof(float) * (size_t)V1 * E, st));
    for (int t = T - 1; t >= 0; --t) {
        const float* c0p = t ? tp.c0 + (long)(t - 1) * NH : nullptr;
        const float* c1p = t ? tp.c1 + (long)(t - 1) * NH : nullptr;
        float* dg1 = tp.DG1 + (long)t * N * 4 * H;
        float* dg2 = tp.DG2 + (long)t * N * 4 * H;
        // language LSTM: dh = carried dh1 + dropout-masked dOUT[:, t]
        if (lstm_cell_backward_launch(N, H, tp.g2 + (long)t * N * 4 * H, c1p, tp.c1 + (long)t * NH, tp.dh1, tp.dOUT + (long)t * H, (long)T * H, 3, (unsigned)t,
                                      seed, p, tp.dc1, dg2, st)) return 1;
        if (sk.dgrad(N, 2 * H, 4 * H, dg2, 4 * H, w.lang_lstm_w_ih, 2 * H, tp.dX2, 2 * H, 0)) return 1;   // [d att_res | d h_att]
        if (sk.dgrad(N, H, 4 * H, dg2, 4 * H, w.lang_lstm_w_hh, H, tp.dh1, H, 0)) return 1;              // carried dh_lang
        // attention: needs a contiguous d att_res
        CAPB_CHECK_CUDA(cudaMemcpy2DAsync(tp.tmpH, sizeof(float) * H, tp.dX2, sizeof(float) * 2 * H, sizeof(float) * H, N, cudaMemcpyDeviceToDevice, st));
        float* datth = tp.DATTH + (long)t * N * A;
        if (attention_backward_launch(B, n, R, A, H, tp.tmpH, tp.alpha + (long)t * N * R, tp.atth + (long)t * N * A, tp.p_att, tp.att_e, w.alpha_w, datth,
                                      tp.d_att_e, tp.d_p_att, G.alpha_w, G.alpha_b, tp.dalpha, st)) return 1;
        // dh_att = carried + d h_att from the language LSTM input + d att_h * W_h2att
        if (add_strided_launch(tp.dh0, tp.dX2 + H, 2 * H, N, H, st)) return 1;
        if (sk.dgrad(N, H, A, datth, A, w.h2att_w, H, tp.dh0, H, 1)) return 1;
        if (lstm_cell_backward_launch(N, H, tp.g1 + (long)t * N * 4 * H, c0p, tp.c0 + (long)t * NH, tp.dh0, nullptr, 0, 0, 0, seed, p, tp.dc0, dg1, st)) return 1;
        // inputs of the attention LSTM: [h_lang_prev | fc' | xt] and h_att_prev
        if (sk.dgrad(N, H, 4 * H, dg1, 4 * H, w.att_lstm_w_ih, E + 2 * H, tp.dh1, H, 1)) return 1;         // += d h_lang_prev
        if (sk.dgrad(N, E, 4 * H, dg1, 4 * H, w.att_lstm_w_ih + 2 * H, E + 2 * H, tp.dxt, E, 0)) return 1;
        if (sk.dgrad(N, H, 4 * H, dg1, 4 * H, w.att_lstm_w_hh, H, tp.dh0, H, 0)) return 1;                // carried dh_att
        if (embed_backward_launch(N, E, tp.tok + (long)t * N, tp.xt + (long)t * N * E, tp.dxt, E, keep_scale, G.embed, st)) return 1;
        e->launches += 12;
    }
    // weight gradients, batched over time (K = T*N)
    const int TN1 = (int)((long)(T - 1) * N);
    const float* DG1s = tp.DG1 + (long)N * 4 * H;     // steps 1..T-1 pair with the previous step's hidden states
    const float* DG2s = tp.DG2 + (long)N * 4 * H;
    int rc = 0;
    rc |= sk.wgrad(4 * H, H, (int)TN, tp.DG2, 4 * H, tp.attres, H, G.lang_lstm_w_ih, 2 * H, 0);
    rc |= sk.wgrad(4 * H, H, (int)TN, tp.DG2, 4 * H, tp.h0, H, G.lang_lstm_w_ih + H, 2 * H, 0);
    rc |= sk.wgrad(4 * H, H, TN1, DG2s, 4 * H, tp.h1, H, G.lang_lstm_w_hh, H, 0);
    rc |= colsum_launch((int)TN, 4 * H, tp.DG2, 4 * H, G.lang_lstm_b_ih, 0, st);
    rc |= colsum_launch((int)TN, 4 * H, tp.DG2, 4 * H, G.lang_lstm_b_hh, 0, st);
    rc |= sk.wgrad(4 * H, H, TN1, DG1s, 4 * H, tp.h1, H, G.att_lstm_w_ih, E + 2 * H, 0);
    rc |= sk.wgrad(4 * H, E, (int)TN, tp.DG1, 4 * H, tp.xt, E, G.att_lstm_w_ih + 2 * H, E + 2 * H, 0);
    rc |= sk.wgrad(4 * H, H, TN1, DG1s, 4 * H, tp.h0, H, G.att_lstm_w_hh, H, 0);
    rc |= colsum_launch((int)TN, 4 * H, tp.DG1, 4 * H, G.att_lstm_b_ih, 0, st);
    rc |= colsum_launch((int)TN, 4 * H, tp.DG1, 4 * H, G.att_lstm_b_hh, 0, st);
    rc |= per_image_sum_launch(T, N, n, 4 * H, tp.DG1, tp.S, st);
    rc |= sk.wgrad(4 * H, H, B, tp.S, 4 * H, tp.fc_e, H, G.att_lstm_w_ih + H, E + 2 * H, 0);               // fc' block
    rc |= sk.dgrad(B, H, 4 * H, tp.S, 4 * H, w.att_lstm_w_ih + H, E + 2 * H, tp.d_fc_e, H, 0);             // d fc'
    rc |= sk.wgrad(A, H, (int)TN, tp.DATTH, A, tp.h0, H, G.h2att_w, H, 0);
    rc |= colsum_launch((int)TN, A, tp.DATTH, A, G.h2att_b, 0, st);
    // prologue
    rc |= att_prologue_backward(e, sk, tp, att, B, R, keep_scale, G, st);
    rc |= relu_dropout_backward_launch((long)B * H, tp.fc_e, tp.d_fc_e, tp.dpre_fc, keep_scale, st);
    rc |= sk.wgrad(H, Ff, B, tp.dpre_fc, H, fc, Ff, G.fc_embed_w, Ff, 0);
    rc |= colsum_launch(B, H, tp.dpre_fc, H, G.fc_embed_b, 0, st);
    e->launches += 27 + (tf32_context_launches(e->tf32) - tf32_l0);     // (incl. the loss's 3) + transposes of the wgmma path
    if (!rc && record_group_event(e->grad_events[1], st)) return 1;
    return rc;
}

// ---- Att2in2 (Att2in2Core, AttModel.py:770-790) ---------------------------------------------------------------------------------------
// One Att2in2 training step: the train-mode forward on the tape (dropout sites 1 att_embed, 2 word embedding, 3 core output, as UpDown),
// the loss, and back-propagation through time.  fc is only handed to the greedy baseline's decode call, which ignores it.
int att2in2_train_step(capb200_engine* e, const float* fc, const float* att, int B, int R, const TrainArgs& ta, const capb200_att2in2_grads* grads,
                       cudaStream_t st) {
    const int n = ta.n, N = B * n, T = ta.T, E = e->E, H = e->H, A = e->A, V1 = e->V1, H5 = 5 * H;
    const float p = ta.p;
    const float keep_scale = 1.0f / (1.0f - p);
    const unsigned long long seed = ta.seed;
    const capb200_weights& w = e->w;
    const long ld_lp = (long)ta.Tl * V1;

    MaxoutTape tp;
    if (carve_tape(&e->tape, &e->tape_bytes, tp, st, [&](MaxoutTape& t, Arena& a) { layout_maxout_tape(t, a, B, R, N, T, E, H, A, V1); })) return 1;
    if (head_train_tape(e, (long)T * N, st)) return 1;
    if (ensure_workspace(e, B, N, R, 1, st)) return 1;
    StepBaseline gb;
    if (start_baseline(e, fc, att, B, R, ta, tp, gb, st)) return 1;
    const Skinny sk = step_gemms(&e->tf32, e->tc, tp, st);
    const long tf32_l0 = tf32_context_launches(e->tf32);

    // ---- train-mode prologue: att_embed (ReLU, dropout site 1, region mask), ctx2att
    nvtxRangePushA("capb200 att2in2 train step: forward on the tape");
    const long BR = (long)B * R, NH = (long)N * H;
    if (att_prologue_forward(e, sk, tp, att, B, R, ta.mask, seed, p, st)) return 1;

    // ---- T steps with the tape
    CAPB_CHECK_CUDA(cudaMemsetAsync(tp.h, 0, sizeof(float) * NH, st));     // slot 0: h = c = 0
    CAPB_CHECK_CUDA(cudaMemsetAsync(tp.c, 0, sizeof(float) * NH, st));
    CAPB_CHECK_CUDA(cudaMemsetAsync(tp.s_tokens, 0, sizeof(int) * N, st));
    for (int t = 0; t < T; ++t) {
        int* tok = tp.tok + (long)t * N;
        if (feed_tokens(ta, tp, N, V1, t, tok, st)) return 1;
        float* xt = tp.xt + (long)t * N * E;
        float* sums = tp.sums + (long)t * N * H5;
        const float* hp = tp.h + (long)t * NH;
        const float* cp = tp.c + (long)t * NH;
        float *h = tp.h + (long)(t + 1) * NH, *c = tp.c + (long)(t + 1) * NH;
        if (embed_relu_dropout_launch(N, E, tok, w.embed, xt, seed, (unsigned)t, p, st)) return 1;
        // attention on the previous hidden state
        float* atth = tp.atth + (long)t * N * A;
        if (sk.lin(hp, H, w.h2att_w, H, w.h2att_b, atth, A, N, A, H, 0)) return 1;
        float* attres = tp.attres + (long)t * NH;
        if (additive_attention_launch(B, n, R, A, H, atth, A, tp.p_att, A, tp.att_e, H, ta.mask, R, w.alpha_w, w.alpha_b, tp.s_att_score,
                                      f32_view(attres, H), st, tp.alpha + (long)t * N * R)) return 1;
        {   // sums = xt i2h^T + h_prev h2h^T + (i2h_b + h2h_b + [0 | a2c_b]), then sums[:, 3H:] += att_res a2c^T
            GemmProblem g; g.M = N; g.N = H5; g.nseg = 2;
            g.seg[0].A = xt; g.seg[0].lda = E; g.seg[0].W = w.i2h_w; g.seg[0].ldw = E; g.seg[0].K = E;
            g.seg[1].A = hp; g.seg[1].lda = H; g.seg[1].W = w.h2h_w; g.seg[1].ldw = H; g.seg[1].K = H;
            g.epi.bias = e->bsum_core;
            g.epi.C = sums; g.epi.ldc = H5;
            if (sk.gates(g)) return 1;
        }
        if (sk.lin(attres, H, w.a2c_w, H, nullptr, sums + 3 * H, H5, N, 2 * H, H, 1)) return 1;
        if (maxout_pointwise_launch(N, H, sums, H5, nullptr, cp, H, c, H, f32_view(h, H), st)) return 1;
        // core output = dropout(h), stored in (n, t) order for the batched logit backward
        float* out = tp.out + (long)t * H;
        if (dropout_copy_launch(h, H, out, (long)T * H, N, H, seed, 3, (unsigned)t, p, st)) return 1;
        const float* lin_in;
        long ld_in;
        if (head_train_forward(e, sk, out, (long)T * H, N, T, t, seed, &lin_in, &ld_in, st)) return 1;
        if (sk.lin(lin_in, ld_in, w.logit_w, H, w.logit_b, ta.logprobs + (long)t * V1, ld_lp, N, V1, H, 0)) return 1;
        if (train_vocab_step(ta, tp, N, V1, t, st)) return 1;
        e->launches += 11;
    }

    // ---- loss, logit backward, back-propagation through time
    nvtxRangePop();
    if (ta.forward_only) return 0;
    CAPB_NVTX("capb200 att2in2 train step: loss, backward through time, weight gradients");
    const long TN = (long)T * N;
    const capb200_att2in2_grads& G = *grads;
    if (loss_and_logit_backward(e, ta, tp, gb, sk, B, N, V1, H, w.logit_w, tp.out, tp.dOUT, G.logit_w, G.logit_b, e->grad_events[0], st)) return 1;
    CAPB_CHECK_CUDA(cudaMemsetAsync(tp.dh, 0, sizeof(float) * NH, st));
    CAPB_CHECK_CUDA(cudaMemsetAsync(tp.dc, 0, sizeof(float) * NH, st));
    CAPB_CHECK_CUDA(cudaMemsetAsync(tp.d_att_e, 0, sizeof(float) * BR * H, st));
    CAPB_CHECK_CUDA(cudaMemsetAsync(tp.d_p_att, 0, sizeof(float) * BR * A, st));
    CAPB_CHECK_CUDA(cudaMemsetAsync(G.alpha_w, 0, sizeof(float) * A, st));
    CAPB_CHECK_CUDA(cudaMemsetAsync(G.alpha_b, 0, sizeof(float), st));
    CAPB_CHECK_CUDA(cudaMemsetAsync(G.embed, 0, sizeof(float) * (size_t)V1 * E, st));
    for (int t = T - 1; t >= 0; --t) {
        const float* sums = tp.sums + (long)t * N * H5;
        float* ds = tp.DS + (long)t * N * H5;
        // cell: dh = carried dh + dropout-masked dOUT[:, t]
        if (maxout_cell_backward_launch(N, H, sums, tp.c + (long)t * NH, tp.c + (long)(t + 1) * NH, tp.dh, tp.dOUT + (long)t * H, (long)T * H, 3,
                                        (unsigned)t, seed, p, tp.dc, ds, st)) return 1;
        if (sk.dgrad(N, E, H5, ds, H5, w.i2h_w, E, tp.dxt, E, 0)) return 1;                     // d xt
        if (sk.dgrad(N, H, H5, ds, H5, w.h2h_w, H, tp.dh, H, 0)) return 1;                      // d h_prev through h2h (the carried dh is consumed)
        if (sk.dgrad(N, H, 2 * H, ds + 3 * H, H5, w.a2c_w, H, tp.d_attres, H, 0)) return 1;     // d att_res: a2c only feeds the candidate pair
        float* datth = tp.DATTH + (long)t * N * A;
        if (attention_backward_launch(B, n, R, A, H, tp.d_attres, tp.alpha + (long)t * N * R, tp.atth + (long)t * N * A, tp.p_att, tp.att_e, w.alpha_w, datth,
                                      tp.d_att_e, tp.d_p_att, G.alpha_w, G.alpha_b, tp.dalpha, st)) return 1;
        if (sk.dgrad(N, H, A, datth, A, w.h2att_w, H, tp.dh, H, 1)) return 1;                   // + d h_prev through h2att
        if (embed_backward_launch(N, E, tp.tok + (long)t * N, tp.xt + (long)t * N * E, tp.dxt, E, keep_scale, G.embed, st)) return 1;
        e->launches += 8;
    }
    // weight gradients, batched over time (K = T*N); h slots 0..T-1 are the previous states h2h and h2att read
    int rc = 0;
    rc |= sk.wgrad(H5, E, (int)TN, tp.DS, H5, tp.xt, E, G.i2h_w, E, 0);
    rc |= sk.wgrad(H5, H, (int)TN, tp.DS, H5, tp.h, H, G.h2h_w, H, 0);
    rc |= sk.wgrad(2 * H, H, (int)TN, tp.DS + 3 * H, H5, tp.attres, H, G.a2c_w, H, 0);
    rc |= colsum_launch((int)TN, H5, tp.DS, H5, G.i2h_b, 0, st);
    rc |= colsum_launch((int)TN, H5, tp.DS, H5, G.h2h_b, 0, st);
    rc |= colsum_launch((int)TN, 2 * H, tp.DS + 3 * H, H5, G.a2c_b, 0, st);
    rc |= sk.wgrad(A, H, (int)TN, tp.DATTH, A, tp.h, H, G.h2att_w, H, 0);
    rc |= colsum_launch((int)TN, A, tp.DATTH, A, G.h2att_b, 0, st);
    rc |= att_prologue_backward(e, sk, tp, att, B, R, keep_scale, G, st);
    e->launches += 11 + (tf32_context_launches(e->tf32) - tf32_l0);     // (incl. the loss's 3)
    if (!rc && record_group_event(e->grad_events[1], st)) return 1;
    return rc;
}

// ---- NewFC (NewFCModel, AttModel.py:904-945; LSTMCore, FCModel.py:13-42) -------------------------------------------------------------
// One NewFC training step.  The core starts from a zero state and first consumes fc_embed(fc) (the image step, AttModel.py:925-927: its
// output is discarded, only (h, c) carries on), then <bos> at t = 0 and the words.  The embedding is a bare nn.Embedding and fc_embed a bare
// nn.Linear (no ReLU, no dropout); the only dropout is site 3 on the core output.  Gradient paths of the image step: h2h(0) is h2h's bias, so
// h2h.bias gets the image step's gradient and h2h.weight does not; i2h gets both the word steps' (input xt) and the image step's (input fc_e);
// fc_embed is reached through the image step only.  The image features are never replicated per row: the image step runs on B rows and
// h / c slot 0 holds its state broadcast to each image's rows.
int newfc_train_step(capb200_engine* e, const float* fc, int B, const TrainArgs& ta, const capb200_newfc_grads* grads, cudaStream_t st) {
    const int n = ta.n, N = B * n, T = ta.T, E = e->E, H = e->H, V1 = e->V1, H5 = 5 * H;
    const int Ff = e->cfg.fc_feat_size;
    const float p = ta.p;
    const unsigned long long seed = ta.seed;
    const capb200_weights& w = e->w;
    const long ld_lp = (long)ta.Tl * V1;

    MaxoutTape tp;
    if (carve_tape(&e->tape, &e->tape_bytes, tp, st, [&](MaxoutTape& t, Arena& a) { layout_newfc_tape(t, a, B, N, T, E, H, V1); })) return 1;
    if (head_train_tape(e, (long)T * N, st)) return 1;
    if (ensure_workspace(e, B, N, 1, 1, st)) return 1;      // R = 1: the region count the greedy baseline's decode call sizes its workspace for
    StepBaseline gb;
    if (start_baseline(e, fc, nullptr, B, 0, ta, tp, gb, st)) return 1;
    const Skinny sk = step_gemms(&e->tf32, e->tc, tp, st);
    const long tf32_l0 = tf32_context_launches(e->tf32);

    // ---- image step on B rows: sums = fc_e i2h^T + (i2h_b + h2h_b), the maxout cell with c_prev = 0
    nvtxRangePushA("capb200 newfc train step: forward on the tape");
    const long NH = (long)N * H;
    if (sk.lin(fc, Ff, w.fc_embed_w, Ff, w.fc_embed_b, tp.fc_e, E, B, E, Ff, 0)) return 1;
    if (sk.lin(tp.fc_e, E, w.i2h_w, E, e->bsum_core, tp.im_sums, H5, B, H5, E, 0)) return 1;
    if (maxout_pointwise_launch(B, H, tp.im_sums, H5, nullptr, nullptr, H, tp.im_c, H, f32_view(tp.im_h, H), st)) return 1;
    iota_div_kernel<<<cdiv(N, 256), 256, 0, st>>>(tp.img_row, N, n);
    CAPB_CHECK_CUDA(cudaGetLastError());
    e->launches += 4;

    // ---- T word steps with the tape
    CAPB_CHECK_CUDA(cudaMemsetAsync(tp.s_tokens, 0, sizeof(int) * N, st));
    for (int t = 0; t < T; ++t) {
        int* tok = tp.tok + (long)t * N;
        if (feed_tokens(ta, tp, N, V1, t, tok, st)) return 1;
        float* xt = tp.xt + (long)t * N * E;
        float* sums = tp.sums + (long)t * N * H5;
        const float* hp = tp.h + (long)t * NH;
        const float* cp = tp.c + (long)t * NH;
        float *h = tp.h + (long)(t + 1) * NH, *c = tp.c + (long)(t + 1) * NH;
        // xt = embed[tok]; at t = 0 the same launch broadcasts the image step's (h, c) into slot 0 of each image's rows (later steps copy no
        // state: H = 0)
        StateCopy s0, s1;
        s0.src = tp.im_h; s0.ld_src = H; s0.dst = f32_view(tp.h, H);
        s1.src = tp.im_c; s1.ld_src = H; s1.dst = f32_view(tp.c, H);
        if (state_gather_embed_launch(N, tok, t == 0 ? tp.img_row : nullptr, w.embed, E, E, 0, f32_view(xt, E), t == 0 ? H : 0,
                                      t == 0 ? 2 : 0, s0, s1, st)) return 1;
        {   // sums = xt i2h^T + h_prev h2h^T + (i2h_b + h2h_b)
            GemmProblem g; g.M = N; g.N = H5; g.nseg = 2;
            g.seg[0].A = xt; g.seg[0].lda = E; g.seg[0].W = w.i2h_w; g.seg[0].ldw = E; g.seg[0].K = E;
            g.seg[1].A = hp; g.seg[1].lda = H; g.seg[1].W = w.h2h_w; g.seg[1].ldw = H; g.seg[1].K = H;
            g.epi.bias = e->bsum_core;
            g.epi.C = sums; g.epi.ldc = H5;
            if (sk.gates(g)) return 1;
        }
        if (maxout_pointwise_launch(N, H, sums, H5, nullptr, cp, H, c, H, f32_view(h, H), st)) return 1;
        // core output = dropout(h) (FCModel.py:40), stored in (n, t) order for the batched logit backward
        float* out = tp.out + (long)t * H;
        if (dropout_copy_launch(h, H, out, (long)T * H, N, H, seed, 3, (unsigned)t, p, st)) return 1;
        const float* lin_in;
        long ld_in;
        if (head_train_forward(e, sk, out, (long)T * H, N, T, t, seed, &lin_in, &ld_in, st)) return 1;
        if (sk.lin(lin_in, ld_in, w.logit_w, H, w.logit_b, ta.logprobs + (long)t * V1, ld_lp, N, V1, H, 0)) return 1;
        if (train_vocab_step(ta, tp, N, V1, t, st)) return 1;
        e->launches += 7;
    }

    // ---- loss, logit backward, back-propagation through time
    nvtxRangePop();
    if (ta.forward_only) return 0;
    CAPB_NVTX("capb200 newfc train step: loss, backward through time, weight gradients");
    const long TN = (long)T * N;
    const capb200_newfc_grads& G = *grads;
    if (loss_and_logit_backward(e, ta, tp, gb, sk, B, N, V1, H, w.logit_w, tp.out, tp.dOUT, G.logit_w, G.logit_b, e->grad_events[0], st)) return 1;
    CAPB_CHECK_CUDA(cudaMemsetAsync(tp.dh, 0, sizeof(float) * NH, st));
    CAPB_CHECK_CUDA(cudaMemsetAsync(tp.dc, 0, sizeof(float) * NH, st));
    CAPB_CHECK_CUDA(cudaMemsetAsync(G.embed, 0, sizeof(float) * (size_t)V1 * E, st));
    for (int t = T - 1; t >= 0; --t) {
        const float* sums = tp.sums + (long)t * N * H5;
        float* ds = tp.DS + (long)t * N * H5;
        // cell: dh = carried dh + dropout-masked dOUT[:, t]
        if (maxout_cell_backward_launch(N, H, sums, tp.c + (long)t * NH, tp.c + (long)(t + 1) * NH, tp.dh, tp.dOUT + (long)t * H, (long)T * H, 3,
                                        (unsigned)t, seed, p, tp.dc, ds, st)) return 1;
        if (sk.dgrad(N, E, H5, ds, H5, w.i2h_w, E, tp.dxt, E, 0)) return 1;                     // d xt
        if (sk.dgrad(N, H, H5, ds, H5, w.h2h_w, H, tp.dh, H, 0)) return 1;                      // d h_prev (the carried dh is consumed)
        if (embed_scatter_launch(N, E, tp.tok + (long)t * N, tp.dxt, E, G.embed, st)) return 1;
        e->launches += 4;
    }
    // the image step: dh / dc carried out of step 0, summed over each image's rows, through the maxout cell (c_prev = 0) on B rows
    int rc = 0;
    rc |= per_image_sum_launch(1, N, n, H, tp.dh, tp.im_dh, st);
    rc |= per_image_sum_launch(1, N, n, H, tp.dc, tp.im_dc, st);
    rc |= maxout_cell_backward_launch(B, H, tp.im_sums, nullptr, tp.im_c, tp.im_dh, nullptr, 0, 0, 0, seed, p, tp.im_dc, tp.im_ds, st);
    // weight gradients, batched over time (K = T*N; h slots 0..T-1 are the previous states h2h reads), plus the image step's terms (K = B)
    rc |= sk.wgrad(H5, E, (int)TN, tp.DS, H5, tp.xt, E, G.i2h_w, E, 0);
    rc |= sk.wgrad(H5, E, B, tp.im_ds, H5, tp.fc_e, E, G.i2h_w, E, 1);
    rc |= sk.wgrad(H5, H, (int)TN, tp.DS, H5, tp.h, H, G.h2h_w, H, 0);
    rc |= colsum_launch((int)TN, H5, tp.DS, H5, G.i2h_b, 0, st);
    rc |= colsum_launch(B, H5, tp.im_ds, H5, G.i2h_b, 1, st);
    rc |= colsum_launch((int)TN, H5, tp.DS, H5, G.h2h_b, 0, st);
    rc |= colsum_launch(B, H5, tp.im_ds, H5, G.h2h_b, 1, st);
    // fc_embed, through the image step's input
    rc |= sk.dgrad(B, E, H5, tp.im_ds, H5, w.i2h_w, E, tp.d_fc_e, E, 0);
    rc |= sk.wgrad(E, Ff, B, tp.d_fc_e, E, fc, Ff, G.fc_embed_w, Ff, 0);
    rc |= colsum_launch(B, E, tp.d_fc_e, E, G.fc_embed_b, 0, st);
    e->launches += 16 + (tf32_context_launches(e->tf32) - tf32_l0);     // (incl. the loss's 3)
    if (!rc && record_group_event(e->grad_events[1], st)) return 1;
    return rc;
}

// the feature checks of a family's training steps: UpDown reads fc and att, Att2in2 att, NewFC fc (and has no regions)
int check_train_feats(const capb200_engine* e, int family, const float* fc, const float* att, int R, const float* att_masks) {
    CAPB_REQUIRE(e->cfg.family == family, "the entry point does not match the engine's family");
    if (family != CAPB200_FAMILY_ATT2IN2) CAPB_REQUIRE(fc != nullptr, "null argument");
    if (family == CAPB200_FAMILY_NEWFC) CAPB_REQUIRE(att_masks == nullptr, "NewFC has no region features: att_masks must be NULL");
    else CAPB_REQUIRE(att != nullptr && R >= 1, "attention features required");
    return 0;
}

// The PPO entry points of UpDown, Att2in2 and NewFC: the family's sampled step `step(ta, stream)` with the PPO criterion, the old policy's
// teacher-forced pass on `old`'s decode path.
template <class Step>
int ppo_entry(capb200_engine* e, capb200_engine* old, int family, const float* fc, const float* att, int B, int R, const capb200_scst_opts* opts,
              const capb200_ppo_opts* ppo, const capb200_cider_table* table, const int* refs, const int* ref_offsets, int L, const void* grads,
              long long* sample_seq, float* sample_logprobs, float* scores, float* loss, float* pg_loss, float* kl_loss, float* clipfrac, cudaStream_t st,
              Step step) {
    if (check_train_ready(e)) return 1;
    CAPB_REQUIRE(opts && table && refs && ref_offsets && grads && sample_seq && sample_logprobs && loss, "null argument");
    CAPB_REQUIRE(R >= 0, "R must be >= 0");
    if (check_train_feats(e, family, fc, att, R, opts->att_masks)) return 1;
    TrainArgs ta;
    if (scst_train_args(B, *opts, table, refs, ref_offsets, L, sample_seq, nullptr, sample_logprobs, nullptr, loss, e->T, &ta)) return 1;
    return run_ppo_step(e, old, ppo, ta, B, scores, pg_loss, kl_loss, clipfrac, st,
                        [&](const capb200_sample_opts* so, const long long* tok, float* lo, void* s) {
                            return capb200_decode_sample(old, fc, att, ta.mask, B, R, so, tok, e->T, nullptr, lo, nullptr, s);
                        },
                        [&] { return step(ta, st); });
}

}  // namespace

// The UpDown, Att2in2 and NewFC entry points take the shared option structs (capb200_scst_opts / capb200_xe_opts) with the same meaning.
extern "C" int capb200_updown_scst_step(capb200_engine* e, const float* fc, const float* att, int B, int R, const capb200_scst_opts* opts,
                                        const capb200_cider_table* table, const int* refs, const int* ref_offsets, int L,
                                        const capb200_updown_grads* grads, long long* sample_seq, long long* greedy_seq, float* sample_logprobs,
                                        float* reward, float* loss, void* stream) {
    if (check_train_ready(e)) return 1;
    CAPB_REQUIRE(opts && table && refs && ref_offsets && grads && sample_seq && sample_logprobs && reward && loss, "null argument");
    if (check_train_feats(e, CAPB200_FAMILY_UPDOWN, fc, att, R, opts->att_masks)) return 1;
    TrainArgs ta;
    if (scst_train_args(B, *opts, table, refs, ref_offsets, L, sample_seq, greedy_seq, sample_logprobs, reward, loss, e->T, &ta)) return 1;
    return run_scst_step(e, opts, grads, ta, fc, sizeof(float) * (size_t)B * e->cfg.fc_feat_size, att, sizeof(float) * (size_t)B * R * e->cfg.att_feat_size,
                         B, R, static_cast<cudaStream_t>(stream),
                         [&](const float* fc_s, const float* att_s, const TrainArgs& t, cudaStream_t s) { return updown_train_step(e, fc_s, att_s, B, R, t, grads, s); });
}

extern "C" int capb200_att2in2_scst_step(capb200_engine* e, const float* fc, const float* att, int B, int R, const capb200_scst_opts* opts,
                                         const capb200_cider_table* table, const int* refs, const int* ref_offsets, int L,
                                         const capb200_att2in2_grads* grads, long long* sample_seq, long long* greedy_seq, float* sample_logprobs,
                                         float* reward, float* loss, void* stream) {
    if (check_train_ready(e)) return 1;
    CAPB_REQUIRE(opts && table && refs && ref_offsets && grads && sample_seq && sample_logprobs && reward && loss, "null argument");
    if (check_train_feats(e, CAPB200_FAMILY_ATT2IN2, fc, att, R, opts->att_masks)) return 1;
    TrainArgs ta;
    if (scst_train_args(B, *opts, table, refs, ref_offsets, L, sample_seq, greedy_seq, sample_logprobs, reward, loss, e->T, &ta)) return 1;
    // the fc features are not read (the greedy baseline's decode call ignores them): not staged
    return run_scst_step(e, opts, grads, ta, fc, 0, att, sizeof(float) * (size_t)B * R * e->cfg.att_feat_size, B, R, static_cast<cudaStream_t>(stream),
                         [&](const float* fc_s, const float* att_s, const TrainArgs& t, cudaStream_t s) { return att2in2_train_step(e, fc_s, att_s, B, R, t, grads, s); });
}

extern "C" int capb200_att2in2_xe_step(capb200_engine* e, const float* fc, const float* att, int B, int R, const capb200_xe_opts* opts,
                                       const long long* labels, const float* masks, int label_cols, const capb200_att2in2_grads* grads, float* logprobs,
                                       float* loss, void* stream) {
    if (check_train_ready(e)) return 1;
    CAPB_REQUIRE(opts && labels && masks && grads && logprobs && loss, "null argument");
    if (check_train_feats(e, CAPB200_FAMILY_ATT2IN2, fc, att, R, opts->att_masks)) return 1;
    TrainArgs ta;
    if (xe_train_args(B, *opts, labels, masks, label_cols, logprobs, loss, e->T, &ta)) return 1;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return run_eager_step(st, [&] { return att2in2_train_step(e, fc, att, B, R, ta, grads, st); });
}

extern "C" int capb200_newfc_scst_step(capb200_engine* e, const float* fc, const float* /*att: NewFC reads the fc features only*/, int B, int R,
                                       const capb200_scst_opts* opts, const capb200_cider_table* table, const int* refs, const int* ref_offsets, int L,
                                       const capb200_newfc_grads* grads, long long* sample_seq, long long* greedy_seq, float* sample_logprobs,
                                       float* reward, float* loss, void* stream) {
    if (check_train_ready(e)) return 1;
    CAPB_REQUIRE(opts && table && refs && ref_offsets && grads && sample_seq && sample_logprobs && reward && loss, "null argument");
    CAPB_REQUIRE(R >= 0, "R must be >= 0");
    if (check_train_feats(e, CAPB200_FAMILY_NEWFC, fc, nullptr, R, opts->att_masks)) return 1;
    TrainArgs ta;
    if (scst_train_args(B, *opts, table, refs, ref_offsets, L, sample_seq, greedy_seq, sample_logprobs, reward, loss, e->T, &ta)) return 1;
    return run_scst_step(e, opts, grads, ta, fc, sizeof(float) * (size_t)B * e->cfg.fc_feat_size, nullptr, 0, B, R, static_cast<cudaStream_t>(stream),
                         [&](const float* fc_s, const float*, const TrainArgs& t, cudaStream_t s) { return newfc_train_step(e, fc_s, B, t, grads, s); });
}

extern "C" int capb200_updown_ppo_step(capb200_engine* e, capb200_engine* old, const float* fc, const float* att, int B, int R, const capb200_scst_opts* opts,
                                       const capb200_ppo_opts* ppo, const capb200_cider_table* table, const int* refs, const int* ref_offsets, int L,
                                       const capb200_updown_grads* grads, long long* sample_seq, float* sample_logprobs, float* scores, float* loss,
                                       float* pg_loss, float* kl_loss, float* clipfrac, void* stream) {
    return ppo_entry(e, old, CAPB200_FAMILY_UPDOWN, fc, att, B, R, opts, ppo, table, refs, ref_offsets, L, grads, sample_seq, sample_logprobs, scores, loss,
                     pg_loss, kl_loss, clipfrac, static_cast<cudaStream_t>(stream),
                     [&](const TrainArgs& ta, cudaStream_t st) { return updown_train_step(e, fc, att, B, R, ta, grads, st); });
}

extern "C" int capb200_att2in2_ppo_step(capb200_engine* e, capb200_engine* old, const float* fc, const float* att, int B, int R, const capb200_scst_opts* opts,
                                        const capb200_ppo_opts* ppo, const capb200_cider_table* table, const int* refs, const int* ref_offsets, int L,
                                        const capb200_att2in2_grads* grads, long long* sample_seq, float* sample_logprobs, float* scores, float* loss,
                                        float* pg_loss, float* kl_loss, float* clipfrac, void* stream) {
    return ppo_entry(e, old, CAPB200_FAMILY_ATT2IN2, fc, att, B, R, opts, ppo, table, refs, ref_offsets, L, grads, sample_seq, sample_logprobs, scores, loss,
                     pg_loss, kl_loss, clipfrac, static_cast<cudaStream_t>(stream),
                     [&](const TrainArgs& ta, cudaStream_t st) { return att2in2_train_step(e, fc, att, B, R, ta, grads, st); });
}

extern "C" int capb200_newfc_ppo_step(capb200_engine* e, capb200_engine* old, const float* fc, const float* /*att: NewFC reads the fc features only*/, int B,
                                      int R, const capb200_scst_opts* opts, const capb200_ppo_opts* ppo, const capb200_cider_table* table, const int* refs,
                                      const int* ref_offsets, int L, const capb200_newfc_grads* grads, long long* sample_seq, float* sample_logprobs,
                                      float* scores, float* loss, float* pg_loss, float* kl_loss, float* clipfrac, void* stream) {
    return ppo_entry(e, old, CAPB200_FAMILY_NEWFC, fc, nullptr, B, R, opts, ppo, table, refs, ref_offsets, L, grads, sample_seq, sample_logprobs, scores, loss,
                     pg_loss, kl_loss, clipfrac, static_cast<cudaStream_t>(stream),
                     [&](const TrainArgs& ta, cudaStream_t st) { return newfc_train_step(e, fc, B, ta, grads, st); });
}

extern "C" int capb200_newfc_xe_step(capb200_engine* e, const float* fc, const float* /*att: NewFC reads the fc features only*/, int B, int R,
                                     const capb200_xe_opts* opts, const long long* labels, const float* masks, int label_cols,
                                     const capb200_newfc_grads* grads, float* logprobs, float* loss, void* stream) {
    if (check_train_ready(e)) return 1;
    CAPB_REQUIRE(opts && labels && masks && grads && logprobs && loss, "null argument");
    CAPB_REQUIRE(R >= 0, "R must be >= 0");
    if (check_train_feats(e, CAPB200_FAMILY_NEWFC, fc, nullptr, R, opts->att_masks)) return 1;
    TrainArgs ta;
    if (xe_train_args(B, *opts, labels, masks, label_cols, logprobs, loss, e->T, &ta)) return 1;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return run_eager_step(st, [&] { return newfc_train_step(e, fc, B, ta, grads, st); });
}

extern "C" int capb200_engine_set_grad_events(capb200_engine* e, void* const* events, int n) { return set_grad_events(e, events, n); }

extern "C" int capb200_updown_xe_step(capb200_engine* e, const float* fc, const float* att, int B, int R, const capb200_xe_opts* opts,
                                      const long long* labels, const float* masks, int label_cols, const capb200_updown_grads* grads, float* logprobs,
                                      float* loss, void* stream) {
    if (check_train_ready(e)) return 1;
    CAPB_REQUIRE(opts && labels && masks && grads && logprobs && loss, "null argument");
    if (check_train_feats(e, CAPB200_FAMILY_UPDOWN, fc, att, R, opts->att_masks)) return 1;
    TrainArgs ta;
    if (xe_train_args(B, *opts, labels, masks, label_cols, logprobs, loss, e->T, &ta)) return 1;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return run_eager_step(st, [&] { return updown_train_step(e, fc, att, B, R, ta, grads, st); });
}

// ---- autograd entry points of UpDown, Att2in2 and NewFC (include/capb200.h: capb200_vjp_opts) ----------------------------------------------
namespace {

template <class Grads, class Step>
int xe_vjp(capb200_engine* e, int family, const float* fc, const float* att, int B, int R, const capb200_xe_opts* opts, const capb200_vjp_opts* vjp,
           const long long* labels, int label_cols, const Grads* grads, float* logprobs, void* stream, Step step) {
    if (check_train_ready(e)) return 1;
    CAPB_REQUIRE(opts && vjp && labels && logprobs && (grads || vjp->forward_only), "null argument");
    if (check_train_feats(e, family, fc, att, R, opts->att_masks)) return 1;
    TrainArgs ta;
    if (xe_train_args(B, *opts, labels, nullptr, label_cols, logprobs, nullptr, e->T, &ta, vjp)) return 1;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return run_vjp_step(e, st, [&] { return step(ta, st); });
}

template <class Grads, class Step>
int scst_vjp(capb200_engine* e, int family, const float* fc, const float* att, int B, int R, const capb200_scst_opts* opts, const capb200_vjp_opts* vjp,
             const Grads* grads, long long* sample_seq, float* sample_logprobs, void* stream, Step step) {
    if (check_train_ready(e)) return 1;
    CAPB_REQUIRE(opts && vjp && sample_seq && sample_logprobs && (grads || vjp->forward_only), "null argument");
    if (check_train_feats(e, family, fc, att, R, opts->att_masks)) return 1;
    TrainArgs ta;
    if (scst_train_args(B, *opts, nullptr, nullptr, nullptr, 0, sample_seq, nullptr, sample_logprobs, nullptr, nullptr, e->T, &ta, vjp)) return 1;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return run_vjp_step(e, st, [&] { return step(ta, st); });
}

}  // namespace

extern "C" int capb200_updown_xe_vjp(capb200_engine* e, const float* fc, const float* att, int B, int R, const capb200_xe_opts* opts,
                                     const capb200_vjp_opts* vjp, const long long* labels, int label_cols, const capb200_updown_grads* grads,
                                     float* logprobs, void* stream) {
    return xe_vjp(e, CAPB200_FAMILY_UPDOWN, fc, att, B, R, opts, vjp, labels, label_cols, grads, logprobs, stream,
                  [&](const TrainArgs& ta, cudaStream_t st) { return updown_train_step(e, fc, att, B, R, ta, grads, st); });
}

extern "C" int capb200_updown_scst_vjp(capb200_engine* e, const float* fc, const float* att, int B, int R, const capb200_scst_opts* opts,
                                       const capb200_vjp_opts* vjp, const capb200_updown_grads* grads, long long* sample_seq, float* sample_logprobs,
                                       void* stream) {
    return scst_vjp(e, CAPB200_FAMILY_UPDOWN, fc, att, B, R, opts, vjp, grads, sample_seq, sample_logprobs, stream,
                    [&](const TrainArgs& ta, cudaStream_t st) { return updown_train_step(e, fc, att, B, R, ta, grads, st); });
}

extern "C" int capb200_att2in2_xe_vjp(capb200_engine* e, const float* fc, const float* att, int B, int R, const capb200_xe_opts* opts,
                                      const capb200_vjp_opts* vjp, const long long* labels, int label_cols, const capb200_att2in2_grads* grads,
                                      float* logprobs, void* stream) {
    return xe_vjp(e, CAPB200_FAMILY_ATT2IN2, fc, att, B, R, opts, vjp, labels, label_cols, grads, logprobs, stream,
                  [&](const TrainArgs& ta, cudaStream_t st) { return att2in2_train_step(e, fc, att, B, R, ta, grads, st); });
}

extern "C" int capb200_att2in2_scst_vjp(capb200_engine* e, const float* fc, const float* att, int B, int R, const capb200_scst_opts* opts,
                                        const capb200_vjp_opts* vjp, const capb200_att2in2_grads* grads, long long* sample_seq, float* sample_logprobs,
                                        void* stream) {
    return scst_vjp(e, CAPB200_FAMILY_ATT2IN2, fc, att, B, R, opts, vjp, grads, sample_seq, sample_logprobs, stream,
                    [&](const TrainArgs& ta, cudaStream_t st) { return att2in2_train_step(e, fc, att, B, R, ta, grads, st); });
}

extern "C" int capb200_newfc_xe_vjp(capb200_engine* e, const float* fc, const float* /*att: NewFC reads the fc features only*/, int B, int R,
                                    const capb200_xe_opts* opts, const capb200_vjp_opts* vjp, const long long* labels, int label_cols,
                                    const capb200_newfc_grads* grads, float* logprobs, void* stream) {
    return xe_vjp(e, CAPB200_FAMILY_NEWFC, fc, nullptr, B, R, opts, vjp, labels, label_cols, grads, logprobs, stream,
                  [&](const TrainArgs& ta, cudaStream_t st) { return newfc_train_step(e, fc, B, ta, grads, st); });
}

extern "C" int capb200_newfc_scst_vjp(capb200_engine* e, const float* fc, const float* /*att: NewFC reads the fc features only*/, int B, int R,
                                      const capb200_scst_opts* opts, const capb200_vjp_opts* vjp, const capb200_newfc_grads* grads, long long* sample_seq,
                                      float* sample_logprobs, void* stream) {
    return scst_vjp(e, CAPB200_FAMILY_NEWFC, fc, nullptr, B, R, opts, vjp, grads, sample_seq, sample_logprobs, stream,
                    [&](const TrainArgs& ta, cudaStream_t st) { return newfc_train_step(e, fc, B, ta, grads, st); });
}

extern "C" {


capb200_cider_table* capb200_cider_table_create(const int* keys, const double* df, long n, double ref_len, void* stream) {
    if (keys == nullptr || df == nullptr || n < 0 || ref_len <= 0) { set_error("bad CIDEr-D table arguments"); return nullptr; }
    CiderTable* t = cider_table_create(keys, df, n, ref_len, static_cast<cudaStream_t>(stream));
    if (t == nullptr) return nullptr;
    capb200_cider_table* h = new capb200_cider_table();
    h->t = t;
    return h;
}

capb200_cider_table* capb200_cider_corpus_table_create(void) {
    CiderTable* t = cider_corpus_table_create();
    if (t == nullptr) return nullptr;
    capb200_cider_table* h = new capb200_cider_table();
    h->t = t;
    return h;
}

int capb200_cider_table_reserve(capb200_cider_table* t, long n_refs, int L) {
    CAPB_REQUIRE(t != nullptr, "null argument");
    return cider_corpus_table_reserve(t->t, n_refs, L);
}

int capb200_cider_table_is_corpus(const capb200_cider_table* t) { return t != nullptr && cider_table_is_corpus(t->t) ? 1 : 0; }

void capb200_cider_table_destroy(capb200_cider_table* t) {
    if (t == nullptr) return;
    cider_table_destroy(t->t);
    delete t;
}

int capb200_self_critical_reward(const capb200_cider_table* t, const long long* sampled, int S, const long long* greedy, int B, int T,
                                 const int* refs, const int* ref_offsets, int L, double* scores, float* reward, void* stream) {
    CAPB_REQUIRE(t != nullptr && sampled && greedy && refs && ref_offsets && scores, "null argument");
    return cider_reward_launch(t->t, sampled, S, greedy, B, T, refs, ref_offsets, L, scores, reward, T, T, static_cast<cudaStream_t>(stream));
}

int capb200_cider_scores(const capb200_cider_table* t, const long long* sampled, int S, int B, int T, const int* refs, const int* ref_offsets,
                         int L, double* scores, float* reward, void* stream) {
    CAPB_REQUIRE(t != nullptr && sampled && refs && ref_offsets && scores, "null argument");
    return cider_reward_launch(t->t, sampled, S, nullptr, B, T, refs, ref_offsets, L, scores, reward, T, T, static_cast<cudaStream_t>(stream));
}

int capb200_bleu4_scores(const long long* sampled, int S, const long long* greedy, int B, int T, const int* refs, const int* ref_offsets, int L,
                         double* scores, void* stream) {
    CAPB_REQUIRE(sampled && refs && ref_offsets && scores, "null argument");
    return bleu_scores_launch(sampled, S, greedy, B, T, refs, ref_offsets, L, scores, static_cast<cudaStream_t>(stream));
}

int capb200_weighted_reward(const capb200_cider_table* t, const capb200_reward_weights* w, const long long* sampled, int S, const long long* greedy,
                            int B, int T, const int* refs, const int* ref_offsets, int L, double* scores, double* bleu_scores, float* reward,
                            void* stream) {
    CAPB_REQUIRE(sampled && refs && ref_offsets && scores, "null argument");
    const double wc = w ? w->cider : 1.0, wb = w ? w->bleu : 0.0;
    return weighted_reward_launch(t ? t->t : nullptr, wc, wb, sampled, S, greedy, B, T, refs, ref_offsets, L, scores, bleu_scores, reward, T, T,
                                  static_cast<cudaStream_t>(stream));
}

int capb200_reward_criterion_forward(const float* logprobs, const long long* seq, const float* reward, int N, int T, int V1, float* loss_mean,
                                     float* loss_rows, float* mask_sum, void* stream) {
    CAPB_REQUIRE(logprobs && seq && reward && N > 0 && T > 0, "bad argument");
    return reward_criterion_fwd_launch(logprobs, (long)T * V1, V1, seq, reward, N, T, loss_mean, loss_rows, mask_sum, static_cast<cudaStream_t>(stream));
}

int capb200_reward_criterion_backward(const long long* seq, const float* reward, int N, int T, int V1, const float* mask_sum, float upstream,
                                      float* grad, void* stream) {
    CAPB_REQUIRE(seq && reward && mask_sum && grad, "null argument");
    return reward_criterion_bwd_launch(seq, reward, N, T, mask_sum, upstream, grad, (long)T * V1, V1, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
