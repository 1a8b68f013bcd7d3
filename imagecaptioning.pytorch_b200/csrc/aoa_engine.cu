// AoANet engine (C ABI capb200_aoa_* in include/capb200.h).
//
// Reference: captioning/models/AoAModel.py
//   _prepare_feature :207-226  att_embed -> 6 AoA refiner layers (:100-126; MultiHeadedDotAttention with project_k_v=1, do_aoa=1
//                              :56-98) -> LayerNorm -> mean pooling (mean_feats) -> ctx2att (H -> 2H = K | V of the decoder attention)
//   AoA_Decoder_Core :163-186  att_lstm(cat[xt, mean + ctx_prev]) -> LayerNorm(h) -> Linear -> 8-head dot attention over the image's
//                              K | V -> GLU(Linear(cat[att, h_att])) = the new context vector, which is also the output and is
//                              carried in state[0][1]; state[1][1] is never touched
// Engine specifics: the mean-feature term of the LSTM gates is contracted once per image (row bias), the word term comes from the
// per-token gate table, the LSTM cell is applied in the GEMM epilogue (tensor-core modes), K | V are indexed per image.
#include <vector>

#include "../../include/capb200.h"
#include "common.cuh"
#include "engine_common.cuh"
#include "kernels.cuh"
#include "train_common.cuh"

using namespace capb200;

struct capb200_aoa_engine : EngineBase {
    capb200_aoa_cfg cfg{};
    capb200_aoa_weights w{};
    int E = 0, H = 0, heads = 0, dk = 0, F = 0;

    float *r_qkv_w[CAPB200_AOA_REFINER_LAYERS] = {}, *r_qkv_b[CAPB200_AOA_REFINER_LAYERS] = {};
    float *bsum = nullptr, *bsum_il = nullptr;
    float* xgate = nullptr;
    long ld_xgate = 0;
    Planes p_att, p_ctx, p_logit, p_ih_x, p_ih_c, p_hh, p_q, p_a2c_a, p_a2c_h;
    Planes pr_qkv[CAPB200_AOA_REFINER_LAYERS], pr_aoa_a[CAPB200_AOA_REFINER_LAYERS], pr_aoa_q[CAPB200_AOA_REFINER_LAYERS];

    Planes in_att;
    Act rx, rln, rqkv, ratt, rt, att_e, mean, p_att_kv, g_mean;     // prologue activations
    Act h0_in, h0_out, ctx_in, ctx_out, xt, gates, qln, qproj, att, t2;   // decoder activations [rows, .]
    float* c0[2] = {nullptr, nullptr};
    long ld_c = 0;
    int core_cur = 0;

    int decode_workspace(int B, int rows, int R, int beam, int rows_per_image, cudaStream_t st) override;
    int decode_prepare(const float* fc, const float* att, const DecodeCtx& c, cudaStream_t st) override;
    int decode_core(int rows, int rpi, const int* tokens, const int* src_row, int t, float* logits, long ld, const DecodeCtx& c, cudaStream_t st) override;
};

namespace {

enum Site { A_ATT = 0, A_CTX, A_GMEAN, A_LSTM, A_Q, A_A2C, A_LOGIT, A_REF /* + 2*l: qkv, aoa */, A_COUNT = A_REF + 2 * CAPB200_AOA_REFINER_LAYERS };

void layout_weights(capb200_aoa_engine* e, Arena& a) {
    const int H = e->H, E = e->E;
    for (int l = 0; l < CAPB200_AOA_REFINER_LAYERS; ++l) { e->r_qkv_w[l] = a.take<float>((long)3 * H * H); e->r_qkv_b[l] = a.take<float>(3 * H); }
    e->bsum = a.take<float>(4 * H);
    e->bsum_il = a.take<float>(4 * H);
    e->ld_xgate = round_up(4 * H, 8);
    e->xgate = a.take<float>((long)e->V1 * e->ld_xgate);
    if (!e->tc) return;
    e->p_att = carve_planes(a, H, e->F);
    e->p_ctx = carve_planes(a, 2 * H, H);
    e->p_logit = carve_planes(a, e->V1, H);
    e->p_ih_x = carve_planes(a, 4 * H, E);
    e->p_ih_c = carve_planes(a, 4 * H, H);
    e->p_hh = carve_planes(a, 4 * H, H);
    e->p_q = carve_planes(a, H, H);
    e->p_a2c_a = carve_planes(a, 2 * H, H);
    e->p_a2c_h = carve_planes(a, 2 * H, H);
    for (int l = 0; l < CAPB200_AOA_REFINER_LAYERS; ++l) {
        e->pr_qkv[l] = carve_planes(a, 3 * H, H);
        e->pr_aoa_a[l] = carve_planes(a, 2 * H, H);
        e->pr_aoa_q[l] = carve_planes(a, 2 * H, H);
    }
}

void layout_workspace(capb200_aoa_engine* e, Arena& a, int B, int rows, int R, int beam) {
    const int H = e->H, E = e->E, T = e->T;
    const bool tc = e->tc;
    const long BR = (long)B * R;
    if (tc) e->in_att = carve_planes(a, BR, e->F);
    e->rx.carve(a, BR, H, false);
    e->rln.carve(a, BR, H, tc);
    e->rqkv.carve(a, BR, 3 * H, false);
    e->ratt.carve(a, BR, H, tc);
    e->rt.carve(a, BR, 2 * H, false);
    e->att_e.carve(a, BR, H, tc);
    e->mean.carve(a, B, H, tc);
    e->p_att_kv.carve(a, BR, 2 * H, false);
    e->g_mean.carve(a, B, 4 * H, false);
    e->h0_in.carve(a, rows, H, tc);
    e->h0_out.carve(a, rows, H, tc);
    e->ctx_in.carve(a, rows, H, tc);
    e->ctx_out.carve(a, rows, H, tc);
    e->xt.carve(a, rows, E, tc);
    e->gates.carve(a, rows, 4 * H, false);
    e->qln.carve(a, rows, H, tc);
    e->qproj.carve(a, rows, H, false);
    e->att.carve(a, rows, H, tc);
    e->t2.carve(a, rows, 2 * H, false);
    e->ld_c = round_up(H, 8);
    for (int i = 0; i < 2; ++i) e->c0[i] = a.take<float>((long)rows * e->ld_c);
    e->carve_head(a, rows);
    e->d.carve(a, B, rows, beam, T);
}

int ensure_workspace(capb200_aoa_engine* e, int B, int rows, int R, int beam, cudaStream_t st) {
    return e->grow(B, rows, R, beam, st, [&](Arena& a, int nB, int nRows, int nR, int nBeam) { layout_workspace(e, a, nB, nRows, nR, nBeam); });
}

int prepare(capb200_aoa_engine* e, const float* att, const float* mask, int B, int R, cudaStream_t st) {
    CAPB_NVTX("capb200 aoa prepare_feature (att_embed, refiner, ctx2att)");
    const int H = e->H, E = e->E, BR = B * R, capBR = e->capB * e->capR;
    const capb200_aoa_weights& w = e->w;
    ActView in; in.f = const_cast<float*>(att); in.ld = e->F;
    if (e->tc) {
        e->launches++;
        if (split_planes_launch(att, e->F, BR, e->F, e->in_att.hi, e->in_att.lo, e->in_att.ld, st)) return 1;
        in.hi = e->in_att.hi; in.lo = e->in_att.lo;
    }
    {
        GemmProblem g;
        g.M = BR; g.N = H; g.nseg = 1;
        g.seg[0] = seg_of(in, w.att_embed_w, e->F, e->p_att, e->F);
        g.seg[0].lda_h = e->in_att.ld;
        g.epi.bias = w.att_embed_b; g.epi.relu = 1;
        g.epi.C = e->rx.v.f; g.epi.ldc = e->rx.v.ld;
        if (e->gemm(A_ATT, g, capBR, st)) return 1;
    }
    if (mask != nullptr) { e->launches++; if (mask_rows_launch(e->rx.v, B, R, H, mask, R, st)) return 1; }
    for (int l = 0; l < CAPB200_AOA_REFINER_LAYERS; ++l) {
        const capb200_aoa_refiner_layer& L = w.refiner[l];
        e->launches++;
        if (layer_norm_launch(BR, H, e->rx.v.f, e->rx.v.ld, L.ln_a, L.ln_b, 1e-6f, e->rln.v, st)) return 1;
        {
            GemmProblem g;
            g.M = BR; g.N = 3 * H; g.nseg = 1;
            g.seg[0] = seg_of(e->rln.v, e->r_qkv_w[l], H, e->pr_qkv[l], H);
            g.epi.bias = e->r_qkv_b[l];
            g.epi.C = e->rqkv.v.f; g.epi.ldc = e->rqkv.v.ld;
            if (e->gemm(A_REF + 2 * l, g, capBR, st)) return 1;
        }
        e->launches++;
        if (enc_self_attention_launch(B, R, e->heads, e->dk, e->rqkv.v.f, e->rqkv.v.f + H, e->rqkv.v.f + 2 * H, e->rqkv.v.ld, mask, R, e->ratt.v, st)) return 1;
        {   // AoA: GLU(Linear(cat[attended, query])) with the normed layer input as the query
            GemmProblem g;
            g.M = BR; g.N = 2 * H; g.nseg = 2;
            g.seg[0] = seg_of(e->ratt.v, L.aoa_w, 2 * H, e->pr_aoa_a[l], H);
            g.seg[1] = seg_of(e->rln.v, L.aoa_w + H, 2 * H, e->pr_aoa_q[l], H);
            g.epi.bias = L.aoa_b;
            g.epi.C = e->rt.v.f; g.epi.ldc = e->rt.v.ld;
            if (e->gemm(A_REF + 2 * l + 1, g, capBR, st)) return 1;
        }
        e->launches++;
        ActView xo = e->rx.v;
        if (glu_launch(BR, H, e->rt.v.f, e->rt.v.ld, e->rx.v.f, e->rx.v.ld, xo, st)) return 1;
    }
    e->launches++;
    if (layer_norm_launch(BR, H, e->rx.v.f, e->rx.v.ld, w.refiner_norm_a, w.refiner_norm_b, 1e-6f, e->att_e.v, st)) return 1;
    e->launches++;
    if (masked_mean_launch(B, R, H, e->att_e.v.f, e->att_e.v.ld, mask, R, e->mean.v, st)) return 1;
    {   // ctx2att: K | V of the decoder attention, per image
        GemmProblem g;
        g.M = BR; g.N = 2 * H; g.nseg = 1;
        g.seg[0] = seg_of(e->att_e.v, w.ctx2att_w, H, e->p_ctx, H);
        g.epi.bias = w.ctx2att_b;
        g.epi.C = e->p_att_kv.v.f; g.epi.ldc = e->p_att_kv.v.ld;
        if (e->gemm(A_CTX, g, capBR, st)) return 1;
    }
    {   // time-invariant gate term: mean_feats * W_ih[:, E:]^T + b_ih + b_hh
        GemmProblem g;
        g.M = B; g.N = 4 * H; g.nseg = 1;
        g.seg[0] = seg_of(e->mean.v, w.att_lstm_w_ih + E, E + H, e->p_ih_c, H);
        g.epi.bias = e->tc ? e->bsum_il : e->bsum;
        g.epi.C = e->g_mean.v.f; g.epi.ldc = e->g_mean.v.ld;
        if (e->gemm(A_GMEAN, g, e->capB, st)) return 1;
    }
    return 0;
}

int core_step(capb200_aoa_engine* e, int rows, int rpi, const int* tokens, const int* src_row, float* logits, long ld_logits, int R,
              const float* mask, cudaStream_t st) {
    const int H = e->H, E = e->E;
    const capb200_aoa_weights& w = e->w;
    StateCopy s0, s1;
    s0.src = e->h0_out.v.f; s0.ld_src = e->h0_out.v.ld; s0.dst = e->h0_in.v;
    s1.src = e->ctx_out.v.f; s1.ld_src = e->ctx_out.v.ld; s1.dst = e->ctx_in.v;
    e->launches++;
    if (state_gather_embed_launch(rows, tokens, src_row, w.embed, E, 0, 1, e->xt.v, H, 2, s0, s1, st)) return 1;
    const int cur = e->core_cur, nxt = cur ^ 1;
    {   // att_lstm gates: ctx_prev and h_att_prev segments + per-image mean term + per-token word term
        GemmProblem g;
        g.M = rows; g.N = 4 * H; g.nseg = 2;
        g.seg[0] = seg_of(e->ctx_in.v, w.att_lstm_w_ih + E, E + H, e->p_ih_c, H);
        g.seg[1] = seg_of(e->h0_in.v, w.att_lstm_w_hh, H, e->p_hh, H);
        g.epi.row_bias = e->g_mean.v.f; g.epi.ld_row_bias = e->g_mean.v.ld; g.epi.rows_per_group = rpi;
        if (e->tc) {
            g.epi.lstm = 1; g.epi.H = H;
            g.epi.c_prev = e->c0[cur]; g.epi.ld_cprev = e->ld_c; g.epi.src_row = src_row;
            g.epi.c_out = e->c0[nxt]; g.epi.ld_cout = e->ld_c;
            g.epi.gather_bias = e->xgate; g.epi.ld_gb = e->ld_xgate; g.epi.gather_idx = tokens;
            g.epi.h_f = e->h0_out.v.f; g.epi.h_hi = e->h0_out.v.hi; g.epi.h_lo = e->h0_out.v.lo; g.epi.ld_h = e->h0_out.v.ld;
        } else {
            g.epi.C = e->gates.v.f; g.epi.ldc = e->gates.v.ld;
        }
        if (e->gemm(A_LSTM, g, e->capRows, st)) return 1;
    }
    if (!e->tc) {
        e->launches++;
        if (lstm_pointwise_launch(rows, H, e->gates.v.f, e->gates.v.ld, src_row, e->c0[cur], e->ld_c, e->c0[nxt], e->ld_c, e->h0_out.v, e->xgate,
                                  e->ld_xgate, tokens, st)) return 1;
    }
    e->core_cur = nxt;
    // multi-head dot attention: LayerNorm(h_att) -> Linear -> heads over the image's K | V (no output layer, no AoA here)
    e->launches++;
    if (layer_norm_launch(rows, H, e->h0_out.v.f, e->h0_out.v.ld, w.attn_norm_a, w.attn_norm_b, 1e-6f, e->qln.v, st)) return 1;
    {
        GemmProblem g;
        g.M = rows; g.N = H; g.nseg = 1;
        g.seg[0] = seg_of(e->qln.v, w.attn_q_w, H, e->p_q, H);
        g.epi.bias = w.attn_q_b;
        g.epi.C = e->qproj.v.f; g.epi.ldc = e->qproj.v.ld;
        if (e->gemm(A_Q, g, e->capRows, st)) return 1;
    }
    e->launches++;
    // AoAModel.py:168 passes (query, value = p_att[..., :H], key = p_att[..., H:]): the first half of ctx2att's output is V, the second K
    if (cross_attention_launch(rows, rpi, e->heads, e->dk, R, e->qproj.v.f, e->qproj.v.ld, e->p_att_kv.v.f + H, e->p_att_kv.v.f, e->p_att_kv.v.ld, mask, R,
                               e->att.v, st)) return 1;
    {   // att2ctx: GLU(Linear(cat[att, h_att]))
        GemmProblem g;
        g.M = rows; g.N = 2 * H; g.nseg = 2;
        g.seg[0] = seg_of(e->att.v, w.att2ctx_w, 2 * H, e->p_a2c_a, H);
        g.seg[1] = seg_of(e->h0_out.v, w.att2ctx_w + H, 2 * H, e->p_a2c_h, H);
        g.epi.bias = w.att2ctx_b;
        g.epi.C = e->t2.v.f; g.epi.ldc = e->t2.v.ld;
        if (e->gemm(A_A2C, g, e->capRows, st)) return 1;
    }
    e->launches++;
    if (glu_launch(rows, H, e->t2.v.f, e->t2.v.ld, nullptr, 0, e->ctx_out.v, st)) return 1;
    ActView x;
    if (e->run_logit_head(e->ctx_out.v, rows, &x, st)) return 1;
    GemmProblem g;
    g.M = rows; g.N = e->V1; g.nseg = 1;
    g.seg[0] = seg_of(x, w.logit_w, H, e->p_logit, H);
    g.epi.bias = w.logit_b;
    g.epi.C = logits; g.epi.ldc = ld_logits;
    return e->gemm(A_LOGIT, g, e->capRows, st);
}

}  // namespace

EngineBase* capb200::engine_base(capb200_aoa_engine* e) { return e; }

int capb200_aoa_engine::decode_workspace(int B, int rows, int R, int beam, int /*rows_per_image*/, cudaStream_t st) {
    return ensure_workspace(this, B, rows, R, beam, st);
}

int capb200_aoa_engine::decode_prepare(const float* /*fc*/, const float* att, const DecodeCtx& c, cudaStream_t st) {
    if (prepare(this, att, c.mask, c.B, c.R, st)) return 1;
    core_cur = 0;
    return 0;
}

int capb200_aoa_engine::decode_core(int rows, int rpi, const int* tokens, const int* src_row, int /*t*/, float* logits, long ld, const DecodeCtx& c,
                                    cudaStream_t st) {
    return core_step(this, rows, rpi, tokens, src_row, logits, ld, c.R, c.mask, st);
}

extern "C" {

capb200_aoa_engine* capb200_aoa_create(const capb200_aoa_cfg* c) {
    if (c == nullptr) { set_error("null cfg"); return nullptr; }
    if (c->heads < 1 || c->rnn_size % c->heads != 0) { set_error("rnn_size must be divisible by the head count"); return nullptr; }
    capb200_aoa_engine* e = create_engine<capb200_aoa_engine>(c->vocab_size, c->seq_length, c->numeric_mode, A_COUNT);
    if (e == nullptr) return nullptr;
    e->cfg = *c;
    e->E = c->input_encoding_size; e->H = c->rnn_size; e->heads = c->heads; e->dk = c->rnn_size / c->heads; e->F = c->att_feat_size;
    e->bind_name = "capb200_aoa_bind_weights";
    e->family = CAPB200_FAMILY_AOA;
    e->graph_family = 9;
    e->grad_groups = 10;
    return e;
}

void capb200_aoa_destroy(capb200_aoa_engine* e) { delete e; }

long capb200_aoa_launch_count(const capb200_aoa_engine* e) { return e ? e->launches : 0; }

int capb200_aoa_bind_weights(capb200_aoa_engine* e, const capb200_aoa_weights* w, void* stream) {
    CAPB_REQUIRE(e != nullptr && w != nullptr, "null argument");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CAPB_REQUIRE(w->embed && w->att_embed_w && w->ctx2att_w && w->att_lstm_w_ih && w->att_lstm_w_hh && w->attn_q_w && w->att2ctx_w && w->logit_w,
                 "missing AoA weights");
    e->w = *w;
    const int H = e->H, E = e->E, V1 = e->V1;
    if (e->alloc_wblock(st, [&](Arena& a) { layout_weights(e, a); })) return 1;
    const long hh = (long)H * H;
    for (int l = 0; l < CAPB200_AOA_REFINER_LAYERS; ++l) {
        const capb200_aoa_refiner_layer& L = w->refiner[l];
        CAPB_CHECK_CUDA(cudaMemcpyAsync(e->r_qkv_w[l], L.q_w, sizeof(float) * hh, cudaMemcpyDeviceToDevice, st));
        CAPB_CHECK_CUDA(cudaMemcpyAsync(e->r_qkv_w[l] + hh, L.k_w, sizeof(float) * hh, cudaMemcpyDeviceToDevice, st));
        CAPB_CHECK_CUDA(cudaMemcpyAsync(e->r_qkv_w[l] + 2 * hh, L.v_w, sizeof(float) * hh, cudaMemcpyDeviceToDevice, st));
        CAPB_CHECK_CUDA(cudaMemcpyAsync(e->r_qkv_b[l], L.q_b, sizeof(float) * H, cudaMemcpyDeviceToDevice, st));
        CAPB_CHECK_CUDA(cudaMemcpyAsync(e->r_qkv_b[l] + H, L.k_b, sizeof(float) * H, cudaMemcpyDeviceToDevice, st));
        CAPB_CHECK_CUDA(cudaMemcpyAsync(e->r_qkv_b[l] + 2 * H, L.v_b, sizeof(float) * H, cudaMemcpyDeviceToDevice, st));
    }
    if (add_vec_launch(w->att_lstm_b_ih, w->att_lstm_b_hh, e->bsum, 4 * H, st) || interleave_gates_launch(e->bsum, e->bsum_il, H, st)) return 1;
    e->launches += 2;
    if (e->tc) {
        int rc = e->pack(w->att_embed_w, e->F, H, e->F, e->p_att, st) | e->pack(w->ctx2att_w, H, 2 * H, H, e->p_ctx, st) |
                 e->pack(w->logit_w, H, V1, H, e->p_logit, st) | e->pack(w->attn_q_w, H, H, H, e->p_q, st) |
                 e->pack(w->att2ctx_w, 2 * H, 2 * H, H, e->p_a2c_a, st) | e->pack(w->att2ctx_w + H, 2 * H, 2 * H, H, e->p_a2c_h, st) |
                 e->pack_gates(w->att_lstm_w_ih, E + H, H, E, e->p_ih_x, st) | e->pack_gates(w->att_lstm_w_ih + E, E + H, H, H, e->p_ih_c, st) |
                 e->pack_gates(w->att_lstm_w_hh, H, H, H, e->p_hh, st);
        for (int l = 0; l < CAPB200_AOA_REFINER_LAYERS; ++l) {
            rc |= e->pack(e->r_qkv_w[l], H, 3 * H, H, e->pr_qkv[l], st) | e->pack(w->refiner[l].aoa_w, 2 * H, 2 * H, H, e->pr_aoa_a[l], st) |
                  e->pack(w->refiner[l].aoa_w + H, 2 * H, 2 * H, H, e->pr_aoa_q[l], st);
        }
        if (rc) return 1;
    }
    // per-token gate table: relu(embed) * W_ih[:, 0:E]^T
    if (build_gate_table(*e, w->embed, E, H, w->att_lstm_w_ih, E + H, e->p_ih_x, e->xgate, e->ld_xgate, st)) return 1;
    return e->finish_bind(st);
}

int capb200_aoa_set_logit_layers(capb200_aoa_engine* e, int logit_layers) {
    CAPB_REQUIRE(e != nullptr, "null engine");
    return e->set_logit_layers(logit_layers, e->H);
}

int capb200_aoa_bind_logit_head(capb200_aoa_engine* e, const float* const* w, const float* const* b, void* stream) {
    CAPB_REQUIRE(e != nullptr, "null engine");
    return e->bind_logit_head(w, b, static_cast<cudaStream_t>(stream));
}

int capb200_aoa_bind_logit_head_grads(capb200_aoa_engine* e, float* const* gw, float* const* gb) {
    CAPB_REQUIRE(e != nullptr, "null engine");
    return e->bind_logit_head_grads(gw, gb);
}

int capb200_aoa_set_logit_dropout(capb200_aoa_engine* e, float p) {
    CAPB_REQUIRE(e != nullptr, "null engine");
    return e->set_logit_dropout(p);
}

int capb200_aoa_decode_beam(capb200_aoa_engine* e, const float* att, const float* mask, int B, int R, const capb200_beam_opts* opts, long long* seq,
                            float* seq_logprobs, long long* done_seq, int* done_len, float* done_p, float* done_raw, void* stream) {
    return decode_beam(e, nullptr, att, mask, B, R, opts, seq, seq_logprobs, done_seq, done_len, done_p, done_raw, static_cast<cudaStream_t>(stream));
}

int capb200_aoa_decode_beam_diverse(capb200_aoa_engine* e, const float* att, const float* mask, int B, int R, const capb200_diverse_opts* opts,
                                    long long* seq, float* seq_logprobs, long long* done_seq, int* done_len, float* done_p, float* done_raw, void* stream) {
    return decode_beam_diverse(e, nullptr, att, mask, B, R, opts, seq, seq_logprobs, done_seq, done_len, done_p, done_raw, static_cast<cudaStream_t>(stream));
}

int capb200_aoa_beam_record_logprobs(capb200_aoa_engine* e, int image, int rank, float* dst, void* stream) {
    return decode_record_logprobs(e, image, rank, dst, static_cast<cudaStream_t>(stream));
}

int capb200_aoa_decode_sample(capb200_aoa_engine* e, const float* att, const float* mask, int B, int R, const capb200_sample_opts* opts,
                              const long long* tokens_in, long ld_tok, long long* seq, float* seq_logprobs, float* picked, void* stream) {
    return decode_sample(e, nullptr, att, mask, B, R, opts, tokens_in, ld_tok, seq, seq_logprobs, picked, static_cast<cudaStream_t>(stream));
}

}  // extern "C"

// =====================================================================================================================
// SCST training step (AoANet)
// =====================================================================================================================
namespace {

constexpr int NL = CAPB200_AOA_REFINER_LAYERS;

struct ATape : StepTape {
    float *x[NL + 1], *ln[NL], *qkv[NL], *ratt[NL], *catd[NL], *t[NL], *g[NL];
    float *att_e, *mean, *kv;
    int* tok;
    float *xt, *x1c, *gates, *c, *h, *qln, *qp, *probs, *att, *t2, *out, *outd;
    float *dOUTD, *D_T2, *D_QP, *DG, *dctx, *dh, *dc, *dX2, *d_qln, *d_hatt, *dxt, *d_x1c, *S, *d_mean, *d_kv, *d_att_e, *d_x, *d_g, *d_t,
        *d_catd, *d_qkv, *d_ln, *dpre, *stats;
};

void layout_atape(ATape& tp, Arena& a, int B, int R, int N, int T, int E, int H, int heads, int V1) {
    const long BR = (long)B * R, TN = (long)T * N;
    for (int l = 0; l <= NL; ++l) tp.x[l] = a.take<float>(BR * H);
    for (int l = 0; l < NL; ++l) {
        tp.ln[l] = a.take<float>(BR * H); tp.qkv[l] = a.take<float>(BR * 3 * H); tp.ratt[l] = a.take<float>(BR * H);
        tp.catd[l] = a.take<float>(BR * 2 * H); tp.t[l] = a.take<float>(BR * 2 * H); tp.g[l] = a.take<float>(BR * H);
    }
    tp.att_e = a.take<float>(BR * H); tp.mean = a.take<float>((long)B * H); tp.kv = a.take<float>(BR * 2 * H);
    tp.tok = a.take<int>(TN);
    tp.xt = a.take<float>(TN * E); tp.x1c = a.take<float>(TN * H); tp.gates = a.take<float>(TN * 4 * H); tp.c = a.take<float>(TN * H);
    tp.h = a.take<float>(TN * H); tp.qln = a.take<float>(TN * H); tp.qp = a.take<float>(TN * H); tp.probs = a.take<float>(TN * heads * R);
    tp.att = a.take<float>(TN * H); tp.t2 = a.take<float>(TN * 2 * H); tp.out = a.take<float>(TN * H); tp.outd = a.take<float>(TN * H);
    tp.layout(a, B, N, TN, V1, (long)B * T * V1);
    tp.dOUTD = a.take<float>(TN * H); tp.D_T2 = a.take<float>(TN * 2 * H); tp.D_QP = a.take<float>(TN * H);
    tp.DG = a.take<float>(TN * 4 * H);
    const long NH = (long)N * H;
    tp.dctx = a.take<float>(NH); tp.dh = a.take<float>(NH); tp.dc = a.take<float>(NH); tp.dX2 = a.take<float>(2 * NH);
    tp.d_qln = a.take<float>(NH); tp.d_hatt = a.take<float>(NH); tp.dxt = a.take<float>((long)N * E); tp.d_x1c = a.take<float>(NH);
    tp.S = a.take<float>((long)B * 4 * H); tp.d_mean = a.take<float>((long)B * H); tp.d_kv = a.take<float>(BR * 2 * H); tp.d_att_e = a.take<float>(BR * H);
    tp.d_x = a.take<float>(BR * H); tp.d_g = a.take<float>(BR * H); tp.d_t = a.take<float>(BR * 2 * H); tp.d_catd = a.take<float>(BR * 2 * H);
    tp.d_qkv = a.take<float>(BR * 3 * H); tp.d_ln = a.take<float>(BR * H); tp.dpre = a.take<float>(BR * H);
    tp.stats = a.take<float>(2 * (BR > N ? BR : N));
}

// the shared arguments (p = drop_prob_lm) and AoANet's other dropout rates
struct AoaTrainArgs : TrainArgs {
    float p_at = 0.f, p_aoa = 0.f, p_sub = 0.f;
    int ctx_drop = 0;
};

// AoANet's own rates (capb200_aoa_xe_opts / capb200_aoa_scst_opts), checked, into `ta`
template <class Opts>
int aoa_rates(const Opts& o, AoaTrainArgs* ta) {
    CAPB_REQUIRE(o.drop_attn >= 0.f && o.drop_attn < 1.f && o.drop_aoa >= 0.f && o.drop_aoa < 1.f && o.drop_sublayer >= 0.f && o.drop_sublayer < 1.f,
                 "dropout rates must be in [0, 1)");
    ta->p_at = o.drop_attn; ta->p_aoa = o.drop_aoa; ta->p_sub = o.drop_sublayer; ta->ctx_drop = o.ctx_drop;
    return 0;
}

// AoANet's options as the shared option structs
capb200_scst_opts shared_opts(const capb200_aoa_scst_opts& o) {
    return {o.sample_n, o.temperature, o.seed, o.drop_prob_lm, o.upstream, o.baseline, o.forced_tokens, o.att_masks, o.keep_rows, o.row_loss, o.sampler,
            o.reward_weights};
}
capb200_xe_opts shared_opts(const capb200_aoa_xe_opts& o) {
    return {o.seq_per_img, o.steps, o.seed, o.drop_prob_lm, o.label_smoothing, o.upstream, o.att_masks, o.ss_prob, o.tokens_used, o.keep_rows, o.row_loss};
}

int aoa_train_step(capb200_aoa_engine* e, const float* att, int B, int R, const AoaTrainArgs& ta, const capb200_aoa_grads* grads, cudaStream_t st) {
    const int n = ta.n, N = B * n, T = ta.T, E = e->E, H = e->H, V1 = e->V1, F = e->F, heads = e->heads, dk = e->dk;
    const float p_lm = ta.p, p_at = ta.p_at, p_aoa = ta.p_aoa, p_sub = ta.p_sub;
    const float p_ctx = ta.ctx_drop ? p_lm : 0.f;
    const float keep_lm = 1.0f / (1.0f - p_lm);
    const unsigned long long seed = ta.seed;
    const capb200_aoa_weights& w = e->w;
    const long BR = (long)B * R, NH = (long)N * H, TN = (long)T * N;
    const long ld_lp = (long)ta.Tl * V1;

    ATape tp;
    if (carve_tape(&e->tape, &e->tape_bytes, tp, st, [&](ATape& t, Arena& a) { layout_atape(t, a, B, R, N, T, E, H, heads, V1); })) return 1;
    if (head_train_tape(e, (long)T * N, st)) return 1;
    // ---- (1) greedy baseline, eval mode: the regular decode path, forked here, enqueued after the prologue
    if (ensure_workspace(e, B, N, R, 1, st)) return 1;         // decode workspace sized before anything is in flight
    StepBaseline gb;
    if (gb.fork(ta, &e->side, &e->ev_fork, &e->ev_join, st)) return 1;
    const Skinny sk = step_gemms(&e->tf32, e->tc, tp, st);
    const long tf32_l0 = tf32_context_launches(e->tf32);

    // ---- (2) train-mode prologue: att_embed (+dropout), six refiner layers, final norm, mean pooling, ctx2att
    nvtxRangePushA("capb200 aoa train step: forward on the tape");
    if (sk.lin(att, F, w.att_embed_w, F, w.att_embed_b, tp.x[0], H, (int)BR, H, F, 0)) return 1;
    if (relu_copy_launch(tp.x[0], BR * H, f32_view(tp.x[0], H), st)) return 1;
    if (dropout_apply_launch(tp.x[0], (int)BR, H, H, seed, 1, 0, p_lm, st)) return 1;
    if (ta.mask != nullptr) {      // pack_wrapper(att_embed): padded regions embed to exactly zero (AoAModel.py:211, AttModel.py:44-49)
        if (mask_rows_launch(f32_view(tp.x[0], H), B, R, H, ta.mask, R, st)) return 1;
        e->launches++;
    }
    for (int l = 0; l < NL; ++l) {
        const capb200_aoa_refiner_layer& Lw = w.refiner[l];
        if (layer_norm_launch((int)BR, H, tp.x[l], H, Lw.ln_a, Lw.ln_b, 1e-6f, f32_view(tp.ln[l], H), st)) return 1;
        if (sk.lin(tp.ln[l], H, e->r_qkv_w[l], H, e->r_qkv_b[l], tp.qkv[l], 3 * H, (int)BR, 3 * H, H, 0)) return 1;
        if (enc_attn_train_launch(B, R, heads, dk, tp.qkv[l], tp.qkv[l] + H, tp.qkv[l] + 2 * H, 3 * H, seed, 10 + l, p_at, tp.ratt[l], H, st, ta.mask, R)) return 1;
        if (cat_dropout_launch((int)BR, H, H, tp.ratt[l], H, tp.ln[l], H, tp.catd[l], 2 * H, seed, 20 + l, 0, p_aoa, st)) return 1;
        if (sk.lin(tp.catd[l], 2 * H, Lw.aoa_w, 2 * H, Lw.aoa_b, tp.t[l], 2 * H, (int)BR, 2 * H, 2 * H, 0)) return 1;
        if (glu_launch((int)BR, H, tp.t[l], 2 * H, nullptr, 0, f32_view(tp.g[l], H), st)) return 1;
        if (add_dropout_launch((int)BR, H, tp.x[l], H, tp.g[l], H, tp.x[l + 1], H, seed, 30 + l, 0, p_sub, st)) return 1;
        e->launches += 9;
    }
    if (layer_norm_launch((int)BR, H, tp.x[NL], H, w.refiner_norm_a, w.refiner_norm_b, 1e-6f, f32_view(tp.att_e, H), st)) return 1;
    if (masked_mean_launch(B, R, H, tp.att_e, H, ta.mask, R, f32_view(tp.mean, H), st)) return 1;
    if (sk.lin(tp.att_e, H, w.ctx2att_w, H, w.ctx2att_b, tp.kv, 2 * H, (int)BR, 2 * H, H, 0)) return 1;
    e->launches += 8;

    // ---- the greedy baseline's ~220 launches are enqueued only now: the side stream forked at the top of the step (it does not wait for the
    // prologue), but the host needs ~0.7 ms to enqueue them, and the main stream should be busy with the prologue meanwhile, not idle
    if (gb.enqueue(B, T, V1, ta.greedy_seq, tp.glp, [&](const capb200_sample_opts* so, const long long* tok, long long* seq, float* lp, void* s) {
            return capb200_aoa_decode_sample(e, att, ta.mask, B, R, so, tok, tok ? T : 0, seq, lp, nullptr, s);
        })) return 1;
    // ---- (3) T sampling steps with the tape
    CAPB_CHECK_CUDA(cudaMemsetAsync(tp.s_tokens, 0, sizeof(int) * N, st));
    for (int t = 0; t < T; ++t) {
        int* tok = tp.tok + (long)t * N;
        if (ta.xe && feed_tokens(ta, tp, N, V1, t, tok, st)) return 1;       // SCST: the fused input launch below reads the previous draw
        float* xt = tp.xt + (long)t * N * E;
        float* x1c = tp.x1c + (long)t * NH;
        float* gates = tp.gates + (long)t * N * 4 * H;
        float *c_t = tp.c + (long)t * NH, *h_t = tp.h + (long)t * NH, *qln = tp.qln + (long)t * NH, *qp = tp.qp + (long)t * NH;
        float *att_t = tp.att + (long)t * NH, *t2 = tp.t2 + (long)t * 2 * NH, *out_t = tp.out + (long)t * NH;
        const float* h_prev = t ? tp.h + (long)(t - 1) * NH : nullptr;
        const float* c_prev = t ? tp.c + (long)(t - 1) * NH : nullptr;
        // one launch: the step's tokens (sampling: the previous step's draw), xt = dropout(relu(embed)), x1c = mean[img] + ctx_drop(previous context)
        if (aoa_step_inputs_launch(N, E, H, n, ta.xe ? tok : tp.s_tokens, ta.xe ? nullptr : tok, w.embed, xt, tp.mean, H, t ? tp.out + (long)(t - 1) * NH : nullptr, x1c,
                                   seed, t, p_lm, p_ctx, st)) return 1;
        {
            GemmProblem g; g.M = N; g.N = 4 * H; g.nseg = 2;
            g.seg[0].A = xt; g.seg[0].lda = E; g.seg[0].W = w.att_lstm_w_ih; g.seg[0].ldw = E + H; g.seg[0].K = E;
            g.seg[1].A = x1c; g.seg[1].lda = H; g.seg[1].W = w.att_lstm_w_ih + E; g.seg[1].ldw = E + H; g.seg[1].K = H;
            if (t) { g.seg[2].A = h_prev; g.seg[2].lda = H; g.seg[2].W = w.att_lstm_w_hh; g.seg[2].ldw = H; g.seg[2].K = H; g.nseg = 3; }
            g.epi.bias = e->bsum; g.epi.C = gates; g.epi.ldc = 4 * H;
            if (sk.gates(g)) return 1;
        }
        if (lstm_ln_launch(N, H, gates, 4 * H, c_prev, H, c_t, H, h_t, H, w.attn_norm_a, w.attn_norm_b, 1e-6f, qln, H, st)) return 1;      // cell + attention.norm
        if (sk.lin(qln, H, w.attn_q_w, H, w.attn_q_b, qp, H, N, H, H, 0)) return 1;
        // AoAModel.py:168 passes (query, value = p_att[..., :H], key = p_att[..., H:])
        if (cross_attn_train_launch(N, n, heads, dk, R, qp, H, tp.kv + H, tp.kv, 2 * H, seed, 5, t, p_at, att_t, H, tp.probs + (long)t * N * heads * R, st,
                                    ta.mask, R)) return 1;
        {
            GemmProblem g; g.M = N; g.N = 2 * H; g.nseg = 2;
            g.seg[0].A = att_t; g.seg[0].lda = H; g.seg[0].W = w.att2ctx_w; g.seg[0].ldw = 2 * H; g.seg[0].K = H;
            g.seg[1].A = h_t; g.seg[1].lda = H; g.seg[1].W = w.att2ctx_w + H; g.seg[1].ldw = 2 * H; g.seg[1].K = H;
            g.epi.bias = w.att2ctx_b; g.epi.C = t2; g.epi.ldc = 2 * H;
            if (sk.gates(g)) return 1;
        }
        float* outd = tp.outd + (long)t * H;                                   // [N][T][H]: batched logit backward
        if (glu_dropout_launch(N, H, t2, 2 * H, out_t, H, outd, (long)T * H, seed, t, p_lm, st)) return 1;
        const float* lin_in;
        long ld_in;
        if (head_train_forward(e, sk, outd, (long)T * H, N, T, t, seed, &lin_in, &ld_in, st)) return 1;
        if (sk.lin(lin_in, ld_in, w.logit_w, H, w.logit_b, ta.logprobs + (long)t * V1, ld_lp, N, V1, H, 0)) return 1;
        if (train_vocab_step(ta, tp, N, V1, t, st)) return 1;
        e->launches += 15;
    }

    // ---- (4) reward and loss, (5) backward through the decoder, starting with the logit layer (group 0)
    nvtxRangePop();
    if (ta.forward_only) return 0;
    CAPB_NVTX("capb200 aoa train step: reward, loss, backward, weight gradients");
    const capb200_aoa_grads& G = *grads;
    if (loss_and_logit_backward(e, ta, tp, gb, sk, B, N, V1, H, w.logit_w, tp.outd, tp.dOUTD, G.logit_w, G.logit_b, e->grad_events[0], st)) return 1;
    CAPB_CHECK_CUDA(cudaMemsetAsync(tp.dctx, 0, sizeof(float) * NH, st));
    CAPB_CHECK_CUDA(cudaMemsetAsync(tp.dh, 0, sizeof(float) * NH, st));
    CAPB_CHECK_CUDA(cudaMemsetAsync(tp.dc, 0, sizeof(float) * NH, st));
    CAPB_CHECK_CUDA(cudaMemsetAsync(tp.d_kv, 0, sizeof(float) * BR * 2 * H, st));
    CAPB_CHECK_CUDA(cudaMemsetAsync(G.embed, 0, sizeof(float) * (size_t)V1 * E, st));
    CAPB_CHECK_CUDA(cudaMemsetAsync(G.attn_norm_a, 0, sizeof(float) * H, st));
    CAPB_CHECK_CUDA(cudaMemsetAsync(G.attn_norm_b, 0, sizeof(float) * H, st));
    for (int t = T - 1; t >= 0; --t) {
        const float* c_prev = t ? tp.c + (long)(t - 1) * NH : nullptr;
        float* d_t2 = tp.D_T2 + (long)t * 2 * NH;
        float* d_qp = tp.D_QP + (long)t * NH;
        float* dg = tp.DG + (long)t * N * 4 * H;
        // d out_t = out_drop-masked logit gradient + what step t+1 received through its (dropped) context input
        if (glu_backward_fused_launch(N, H, tp.t2 + (long)t * 2 * NH, 2 * H, tp.dOUTD + (long)t * H, (long)T * H, tp.dctx, d_t2, 2 * H, seed, t, p_lm, st)) return 1;
        if (sk.dgrad(N, 2 * H, 2 * H, d_t2, 2 * H, w.att2ctx_w, 2 * H, tp.dX2, 2 * H, 0)) return 1;             // [d att | d h_att]
        // attention: d att is the first half of dX2's rows (pitch 2H)
        if (cross_attn_backward_launch(B, n, heads, dk, R, tp.qp + (long)t * NH, H, tp.kv + H, tp.kv, 2 * H, seed, 5, t, p_at, tp.probs + (long)t * N * heads * R,
                                       tp.dX2, 2 * H, d_qp, H, tp.d_kv + H, tp.d_kv, 2 * H, st)) return 1;
        if (sk.dgrad(N, H, H, d_qp, H, w.attn_q_w, H, tp.d_qln, H, 0)) return 1;
        // d h_att = carried (from W_hh of step t+1) + att2ctx's h_att half + through the query LayerNorm
        if (ln_backward_launch(N, H, tp.h + (long)t * NH, H, w.attn_norm_a, tp.d_qln, H, 1e-6f, tp.d_hatt, H, 0, tp.stats, G.attn_norm_a, G.attn_norm_b, 1, st,
                               tp.dX2 + H, 2 * H, tp.dh, H)) return 1;
        if (lstm_cell_backward_launch(N, H, tp.gates + (long)t * N * 4 * H, c_prev, tp.c + (long)t * NH, tp.d_hatt, nullptr, 0, 0, 0, seed, 0.f, tp.dc, dg, st)) return 1;
        if (sk.dgrad(N, E, 4 * H, dg, 4 * H, w.att_lstm_w_ih, E + H, tp.dxt, E, 0)) return 1;
        if (sk.dgrad(N, H, 4 * H, dg, 4 * H, w.att_lstm_w_ih + E, E + H, tp.d_x1c, H, 0)) return 1;
        if (sk.dgrad(N, H, 4 * H, dg, 4 * H, w.att_lstm_w_hh, H, tp.dh, H, 0)) return 1;                             // carried to step t-1
        if (embed_backward_launch(N, E, tp.tok + (long)t * N, tp.xt + (long)t * N * E, tp.dxt, E, keep_lm, G.embed, st)) return 1;
        // the context input of step t is ctx_drop(out_{t-1}): its gradient flows to out_{t-1}
        if (t > 0 && dropout_copy_launch(tp.d_x1c, H, tp.dctx, H, N, H, seed, 4, (unsigned)t, p_ctx, st)) return 1;
        e->launches += 17;
    }
    // weight gradients batched over time (K = T*N rows)
    const int TN1 = (int)((long)(T - 1) * N);
    int rc = 0;
    rc |= sk.wgrad(2 * H, H, (int)TN, tp.D_T2, 2 * H, tp.att, H, G.att2ctx_w, 2 * H, 0);
    rc |= sk.wgrad(2 * H, H, (int)TN, tp.D_T2, 2 * H, tp.h, H, G.att2ctx_w + H, 2 * H, 0);
    rc |= colsum_launch((int)TN, 2 * H, tp.D_T2, 2 * H, G.att2ctx_b, 0, st);
    rc |= sk.wgrad(H, H, (int)TN, tp.D_QP, H, tp.qln, H, G.attn_q_w, H, 0);
    rc |= colsum_launch((int)TN, H, tp.D_QP, H, G.attn_q_b, 0, st);
    rc |= sk.wgrad(4 * H, E, (int)TN, tp.DG, 4 * H, tp.xt, E, G.att_lstm_w_ih, E + H, 0);
    rc |= sk.wgrad(4 * H, H, (int)TN, tp.DG, 4 * H, tp.x1c, H, G.att_lstm_w_ih + E, E + H, 0);
    if (TN1 > 0) rc |= sk.wgrad(4 * H, H, TN1, tp.DG + (long)N * 4 * H, 4 * H, tp.h, H, G.att_lstm_w_hh, H, 0);
    else CAPB_CHECK_CUDA(cudaMemsetAsync(G.att_lstm_w_hh, 0, sizeof(float) * 4 * H * H, st));
    rc |= colsum_launch((int)TN, 4 * H, tp.DG, 4 * H, G.att_lstm_b_ih, 0, st);
    rc |= colsum_launch((int)TN, 4 * H, tp.DG, 4 * H, G.att_lstm_b_hh, 0, st);
    // mean_feats enters every step's gate input: d mean[img] = (sum over steps and the image's rows of d gates) * W_ih[:, E:]
    rc |= per_image_sum_launch(T, N, n, 4 * H, tp.DG, tp.S, st);
    rc |= sk.dgrad(B, H, 4 * H, tp.S, 4 * H, w.att_lstm_w_ih + E, E + H, tp.d_mean, H, 0);
    if (rc) return 1;
    if (record_group_event(e->grad_events[1], st)) return 1;                                        // decoder + embed

    // ---- (6) backward through the prologue
    rc |= sk.dgrad((int)BR, H, 2 * H, tp.d_kv, 2 * H, w.ctx2att_w, H, tp.d_att_e, H, 0);
    rc |= sk.wgrad(2 * H, H, (int)BR, tp.d_kv, 2 * H, tp.att_e, H, G.ctx2att_w, H, 0);
    rc |= colsum_launch((int)BR, 2 * H, tp.d_kv, 2 * H, G.ctx2att_b, 0, st);
    rc |= mean_backward_launch(B, R, H, tp.d_mean, H, tp.d_att_e, H, st, ta.mask, R);
    rc |= ln_backward_launch((int)BR, H, tp.x[NL], H, w.refiner_norm_a, tp.d_att_e, H, 1e-6f, tp.d_x, H, 0, tp.stats, G.refiner_norm_a, G.refiner_norm_b, 0, st);
    if (rc) return 1;
    if (record_group_event(e->grad_events[2], st)) return 1;                                        // ctx2att + refiner.norm
    for (int l = NL - 1; l >= 0; --l) {
        const capb200_aoa_refiner_layer& Lw = w.refiner[l];
        const capb200_aoa_refiner_layer_grads& Lg = G.refiner[l];
        // x[l+1] = x[l] + dropout(g): d_x carries to x[l] unchanged; d g = d_x * mask
        rc |= dropout_copy_launch(tp.d_x, H, tp.d_g, H, (int)BR, H, seed, 30 + l, 0, p_sub, st);
        rc |= glu_backward_launch((int)BR, H, tp.t[l], 2 * H, tp.d_g, H, tp.d_t, 2 * H, st);
        rc |= sk.wgrad(2 * H, 2 * H, (int)BR, tp.d_t, 2 * H, tp.catd[l], 2 * H, Lg.aoa_w, 2 * H, 0);
        rc |= colsum_launch((int)BR, 2 * H, tp.d_t, 2 * H, Lg.aoa_b, 0, st);
        rc |= sk.dgrad((int)BR, 2 * H, 2 * H, tp.d_t, 2 * H, Lw.aoa_w, 2 * H, tp.d_catd, 2 * H, 0);
        rc |= dropout_apply_launch(tp.d_catd, (int)BR, 2 * H, 2 * H, seed, 20 + l, 0, p_aoa, st);               // [d attended | d ln (query half)]
        // self-attention backward needs a contiguous d attended
        CAPB_CHECK_CUDA(cudaMemcpy2DAsync(tp.d_g, sizeof(float) * H, tp.d_catd, sizeof(float) * 2 * H, sizeof(float) * H, BR, cudaMemcpyDeviceToDevice, st));
        rc |= enc_attn_backward_launch(B, R, heads, dk, tp.qkv[l], tp.qkv[l] + H, tp.qkv[l] + 2 * H, 3 * H, seed, 10 + l, p_at, tp.d_g, H, tp.d_qkv, tp.d_qkv + H,
                                       tp.d_qkv + 2 * H, 3 * H, st, ta.mask, R);
        rc |= qkv_grads(sk, (int)BR, H, tp.d_qkv, tp.ln[l], Lg, nullptr, st);     // (counted in the layer's launches)
        // d ln = query half of the AoA input + through the packed q|k|v projection
        CAPB_CHECK_CUDA(cudaMemcpy2DAsync(tp.d_ln, sizeof(float) * H, tp.d_catd + H, sizeof(float) * 2 * H, sizeof(float) * H, BR, cudaMemcpyDeviceToDevice, st));
        rc |= sk.dgrad((int)BR, H, 3 * H, tp.d_qkv, 3 * H, e->r_qkv_w[l], H, tp.d_ln, H, 1);
        rc |= ln_backward_launch((int)BR, H, tp.x[l], H, Lw.ln_a, tp.d_ln, H, 1e-6f, tp.d_x, H, 1, tp.stats, Lg.ln_a, Lg.ln_b, 0, st);
        if (rc) return 1;
        if (record_group_event(e->grad_events[3 + (NL - 1 - l)], st)) return 1;                     // refiner layer l (layers finish 5 -> 0)
        e->launches += 22;
    }
    rc |= relu_dropout_backward_launch(BR * H, tp.x[0], tp.d_x, tp.dpre, keep_lm, st);
    rc |= sk.wgrad(H, F, (int)BR, tp.dpre, H, att, F, G.att_embed_w, F, 0);
    rc |= colsum_launch((int)BR, H, tp.dpre, H, G.att_embed_b, 0, st);
    e->launches += tf32_context_launches(e->tf32) - tf32_l0;
    if (!rc && record_group_event(e->grad_events[9], st)) return 1;                                 // att_embed
    return rc;
}

}  // namespace

extern "C" int capb200_aoa_scst_step(capb200_aoa_engine* e, const float* att, int B, int R, const capb200_aoa_scst_opts* opts,
                                     const capb200_cider_table* table, const int* refs, const int* ref_offsets, int L, const capb200_aoa_grads* grads,
                                     long long* sample_seq, long long* greedy_seq, float* sample_logprobs, float* reward, float* loss, void* stream) {
    if (check_train_ready(e)) return 1;
    CAPB_REQUIRE(opts && att && table && refs && ref_offsets && grads && sample_seq && sample_logprobs && reward && loss, "null argument");
    CAPB_REQUIRE(R >= 1, "attention features required");
    AoaTrainArgs ta;
    if (aoa_rates(*opts, &ta) ||
        scst_train_args(B, shared_opts(*opts), table, refs, ref_offsets, L, sample_seq, greedy_seq, sample_logprobs, reward, loss, e->T, &ta)) return 1;
    return run_scst_step(e, opts, grads, ta, nullptr, 0, att, sizeof(float) * (size_t)B * R * e->F, B, R, static_cast<cudaStream_t>(stream),
                         [&](const float*, const float* att_s, const AoaTrainArgs& t, cudaStream_t s) { return aoa_train_step(e, att_s, B, R, t, grads, s); });
}

// PPO (include/capb200.h: capb200_ppo_opts): the sampled step with the PPO criterion; the old policy's teacher-forced pass runs on `old`.
extern "C" int capb200_aoa_ppo_step(capb200_aoa_engine* e, capb200_aoa_engine* old, const float* att, int B, int R, const capb200_aoa_scst_opts* opts,
                                    const capb200_ppo_opts* ppo, const capb200_cider_table* table, const int* refs, const int* ref_offsets, int L,
                                    const capb200_aoa_grads* grads, long long* sample_seq, float* sample_logprobs, float* scores, float* loss, float* pg_loss,
                                    float* kl_loss, float* clipfrac, void* stream) {
    if (check_train_ready(e)) return 1;
    CAPB_REQUIRE(opts && att && table && refs && ref_offsets && grads && sample_seq && sample_logprobs && loss, "null argument");
    CAPB_REQUIRE(R >= 1, "attention features required");
    AoaTrainArgs ta;
    if (aoa_rates(*opts, &ta) ||
        scst_train_args(B, shared_opts(*opts), table, refs, ref_offsets, L, sample_seq, nullptr, sample_logprobs, nullptr, loss, e->T, &ta)) return 1;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return run_ppo_step(e, old, ppo, ta, B, scores, pg_loss, kl_loss, clipfrac, st,
                        [&](const capb200_sample_opts* so, const long long* tok, float* lo, void* s) {
                            return capb200_aoa_decode_sample(old, att, ta.mask, B, R, so, tok, e->T, nullptr, lo, nullptr, s);
                        },
                        [&] { return aoa_train_step(e, att, B, R, ta, grads, st); });
}

extern "C" int capb200_aoa_set_grad_events(capb200_aoa_engine* e, void* const* events, int n) { return set_grad_events(e, events, n); }

extern "C" int capb200_aoa_xe_step(capb200_aoa_engine* e, const float* att, int B, int R, const capb200_aoa_xe_opts* opts, const long long* labels,
                                   const float* masks, int label_cols, const capb200_aoa_grads* grads, float* logprobs, float* loss, void* stream) {
    if (check_train_ready(e)) return 1;
    CAPB_REQUIRE(opts && att && labels && masks && grads && logprobs && loss, "null argument");
    CAPB_REQUIRE(R >= 1, "attention features required");
    AoaTrainArgs ta;
    if (aoa_rates(*opts, &ta) || xe_train_args(B, shared_opts(*opts), labels, masks, label_cols, logprobs, loss, e->T, &ta)) return 1;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return run_eager_step(st, [&] { return aoa_train_step(e, att, B, R, ta, grads, st); });
}

// The autograd entry points (include/capb200.h: capb200_vjp_opts) on AoANet's option structs.
extern "C" int capb200_aoa_xe_vjp(capb200_aoa_engine* e, const float* att, int B, int R, const capb200_aoa_xe_opts* opts, const capb200_vjp_opts* vjp,
                                  const long long* labels, int label_cols, const capb200_aoa_grads* grads, float* logprobs, void* stream) {
    if (check_train_ready(e)) return 1;
    CAPB_REQUIRE(opts && vjp && att && labels && logprobs && (grads || vjp->forward_only), "null argument");
    CAPB_REQUIRE(R >= 1, "attention features required");
    AoaTrainArgs ta;
    if (aoa_rates(*opts, &ta) || xe_train_args(B, shared_opts(*opts), labels, nullptr, label_cols, logprobs, nullptr, e->T, &ta, vjp)) return 1;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return run_vjp_step(e, st, [&] { return aoa_train_step(e, att, B, R, ta, grads, st); });
}

extern "C" int capb200_aoa_scst_vjp(capb200_aoa_engine* e, const float* att, int B, int R, const capb200_aoa_scst_opts* opts, const capb200_vjp_opts* vjp,
                                    const capb200_aoa_grads* grads, long long* sample_seq, float* sample_logprobs, void* stream) {
    if (check_train_ready(e)) return 1;
    CAPB_REQUIRE(opts && vjp && att && sample_seq && sample_logprobs && (grads || vjp->forward_only), "null argument");
    CAPB_REQUIRE(R >= 1, "attention features required");
    capb200_scst_opts shared = shared_opts(*opts);
    shared.reward_weights = nullptr;     // no reward runs under the autograd entry points
    AoaTrainArgs ta;
    if (aoa_rates(*opts, &ta) ||
        scst_train_args(B, shared, nullptr, nullptr, nullptr, 0, sample_seq, nullptr, sample_logprobs, nullptr, nullptr, e->T, &ta, vjp)) return 1;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return run_vjp_step(e, st, [&] { return aoa_train_step(e, att, B, R, ta, grads, st); });
}
