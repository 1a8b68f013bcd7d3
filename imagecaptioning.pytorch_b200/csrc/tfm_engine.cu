// Transformer captioner engine (C ABI capb200_tfm_* in include/capb200.h).
//
// Reference: captioning/models/TransformerModel.py -- _prepare_feature :305-338 (att_embed + N_enc pre-norm encoder layers),
// core :351-363 (the reference re-runs the whole decoder over all t tokens every step; here every layer keeps a K/V cache and a
// step touches one token per row -- 20 token-layers instead of 210 per caption, same results since the decoder mask is causal),
// Generator :50-57.  Beam search / sampling bookkeeping is the shared driver of engine_common.cuh; a beam row reads its
// ancestors' cache entries through the search history, so the cache is never reordered by parent beam (the reference reorders
// its token history, CaptionModel.py:105-108).
#include <vector>

#include "../../include/capb200.h"
#include "common.cuh"
#include "engine_common.cuh"
#include "train_common.cuh"
#include "kernels.cuh"

using namespace capb200;

namespace capb200 {
const char* last_error_cstr();
}

struct capb200_tfm_engine : EngineBase {
    capb200_tfm_cfg cfg{};
    capb200_tfm_weights w{};
    int D = 0, Dff = 0, H = 0, dk = 0, NE = 0, ND = 0, F = 0;

    // bind-time (in the weight block): concatenated projections and their split planes
    float *enc_qkv_w[CAPB200_TFM_MAX_LAYERS] = {}, *enc_qkv_b[CAPB200_TFM_MAX_LAYERS] = {};
    float *dec_qkv_w[CAPB200_TFM_MAX_LAYERS] = {}, *dec_qkv_b[CAPB200_TFM_MAX_LAYERS] = {};
    float *dec_skv_w[CAPB200_TFM_MAX_LAYERS] = {}, *dec_skv_b[CAPB200_TFM_MAX_LAYERS] = {};
    Planes p_att, p_gen;
    Planes pe_qkv[CAPB200_TFM_MAX_LAYERS], pe_o[CAPB200_TFM_MAX_LAYERS], pe_w1[CAPB200_TFM_MAX_LAYERS], pe_w2[CAPB200_TFM_MAX_LAYERS];
    Planes pd_qkv[CAPB200_TFM_MAX_LAYERS], pd_o[CAPB200_TFM_MAX_LAYERS], pd_qs[CAPB200_TFM_MAX_LAYERS], pd_skv[CAPB200_TFM_MAX_LAYERS],
        pd_os[CAPB200_TFM_MAX_LAYERS], pd_w1[CAPB200_TFM_MAX_LAYERS], pd_w2[CAPB200_TFM_MAX_LAYERS];

    // workspace
    Planes in_att;
    Act ex, eln, eqkv, eatt, eh, mem;            // encoder activations [B*R, .]
    float* skv[CAPB200_TFM_MAX_LAYERS] = {};     // per decoder layer [B*R, 2D]: K | V of the memory
    Act x, ln, qkv, att, qs, hh;                 // decoder activations [rows, .]
    float *kc[CAPB200_TFM_MAX_LAYERS] = {}, *vc[CAPB200_TFM_MAX_LAYERS] = {};   // [T][rows][D]
    long cache_step_stride = 0;

    int decode_workspace(int B, int rows, int R, int beam, int rows_per_image, cudaStream_t st) override;
    int decode_prepare(const float* fc, const float* att, const DecodeCtx& c, cudaStream_t st) override;
    int decode_core(int rows, int rpi, const int* tokens, const int* src_row, int t, float* logits, long ld, const DecodeCtx& c, cudaStream_t st) override;
};

namespace {

enum Site { S_ATT = 0, S_GEN = 1, S_ENC = 2 /* + 4*l: qkv,o,w1,w2 */, S_SKV = 2 + 4 * CAPB200_TFM_MAX_LAYERS /* + l */,
            S_DEC = S_SKV + CAPB200_TFM_MAX_LAYERS /* + 6*l: qkv,o,qs,os,w1,w2 */, S_COUNT = S_DEC + 6 * CAPB200_TFM_MAX_LAYERS };

// y = f32_view(x * W^T + b) (+ residual); x given as an ActView, W as fp32 pointer + planes
int linear(capb200_tfm_engine* e, int site, const ActView& x, int M, int K, const float* w, const Planes& wp, const float* b, int N, ActView out,
           bool relu, const float* residual, long ld_res, int plan_rows, cudaStream_t st) {
    GemmProblem g;
    g.M = M; g.N = N; g.nseg = 1;
    g.seg[0] = seg_of(x, w, K, wp, K);
    g.epi.bias = b; g.epi.relu = relu ? 1 : 0;
    g.epi.residual = residual; g.epi.ld_res = ld_res;
    g.epi.C = out.f; g.epi.ldc = out.ld; g.epi.C_hi = out.hi; g.epi.C_lo = out.lo; g.epi.ldcs = out.ld;
    return e->gemm(site, g, plan_rows, st);
}

void layout_weights(capb200_tfm_engine* e, Arena& a) {
    const int D = e->D, Dff = e->Dff;
    for (int l = 0; l < e->NE; ++l) { e->enc_qkv_w[l] = a.take<float>((long)3 * D * D); e->enc_qkv_b[l] = a.take<float>(3 * D); }
    for (int l = 0; l < e->ND; ++l) {
        e->dec_qkv_w[l] = a.take<float>((long)3 * D * D); e->dec_qkv_b[l] = a.take<float>(3 * D);
        e->dec_skv_w[l] = a.take<float>((long)2 * D * D); e->dec_skv_b[l] = a.take<float>(2 * D);
    }
    if (!e->tc) return;
    e->p_att = carve_planes(a, D, e->F);
    e->p_gen = carve_planes(a, e->V1, D);
    for (int l = 0; l < e->NE; ++l) {
        e->pe_qkv[l] = carve_planes(a, 3 * D, D); e->pe_o[l] = carve_planes(a, D, D);
        e->pe_w1[l] = carve_planes(a, Dff, D); e->pe_w2[l] = carve_planes(a, D, Dff);
    }
    for (int l = 0; l < e->ND; ++l) {
        e->pd_qkv[l] = carve_planes(a, 3 * D, D); e->pd_o[l] = carve_planes(a, D, D); e->pd_qs[l] = carve_planes(a, D, D);
        e->pd_skv[l] = carve_planes(a, 2 * D, D); e->pd_os[l] = carve_planes(a, D, D);
        e->pd_w1[l] = carve_planes(a, Dff, D); e->pd_w2[l] = carve_planes(a, D, Dff);
    }
}

void layout_workspace(capb200_tfm_engine* e, Arena& a, int B, int rows, int R, int beam) {
    const int D = e->D, Dff = e->Dff, T = e->T;
    const bool tc = e->tc;
    const long BR = (long)B * R;
    if (tc) e->in_att = carve_planes(a, BR, e->F);
    e->ex.carve(a, BR, D, false);
    e->eln.carve(a, BR, D, tc);
    e->eqkv.carve(a, BR, 3 * D, false);
    e->eatt.carve(a, BR, D, tc);
    e->eh.carve(a, BR, Dff, tc);
    e->mem.carve(a, BR, D, tc);
    for (int l = 0; l < e->ND; ++l) e->skv[l] = a.take<float>(BR * 2 * D);
    e->x.carve(a, rows, D, false);
    e->ln.carve(a, rows, D, tc);
    e->qkv.carve(a, rows, 3 * D, false);
    e->att.carve(a, rows, D, tc);
    e->qs.carve(a, rows, D, false);
    e->hh.carve(a, rows, Dff, tc);
    e->cache_step_stride = (long)rows * D;
    for (int l = 0; l < e->ND; ++l) {
        e->kc[l] = a.take<float>((long)(T + 1) * rows * D);      // T + 1 positions: teacher forcing feeds bos + T labels
        e->vc[l] = a.take<float>((long)(T + 1) * rows * D);
    }
    e->d.carve(a, B, rows, beam, T);
}

int ensure_workspace(capb200_tfm_engine* e, int B, int rows, int R, int beam, cudaStream_t st) {
    return e->grow(B, rows, R, beam, st, [&](Arena& a, int nB, int nRows, int nR, int nBeam) { layout_workspace(e, a, nB, nRows, nR, nBeam); });
}

// the split planes of a contiguous weight [rows, cols]
int pack(capb200_tfm_engine* e, const float* w, int rows, int cols, const Planes& p, cudaStream_t st) { return e->pack(w, cols, rows, cols, p, st); }

int concat_rows(float* dst, const float* a, const float* b, const float* c, long n_each, cudaStream_t st) {
    CAPB_CHECK_CUDA(cudaMemcpyAsync(dst, a, sizeof(float) * n_each, cudaMemcpyDeviceToDevice, st));
    CAPB_CHECK_CUDA(cudaMemcpyAsync(dst + n_each, b, sizeof(float) * n_each, cudaMemcpyDeviceToDevice, st));
    if (c) CAPB_CHECK_CUDA(cudaMemcpyAsync(dst + 2 * n_each, c, sizeof(float) * n_each, cudaMemcpyDeviceToDevice, st));
    return 0;
}

// _prepare_feature: att_embed (+ReLU), N_enc pre-norm encoder layers, final LayerNorm, then K/V of every decoder layer's src_attn
int prepare(capb200_tfm_engine* e, const float* att, const float* mask, int B, int R, cudaStream_t st) {
    const int D = e->D, Dff = e->Dff, BR = B * R, capBR = e->capB * e->capR;
    const capb200_tfm_weights& w = e->w;
    ActView in; in.f = const_cast<float*>(att); in.ld = e->F;
    if (e->tc) {
        e->launches++;
        if (split_planes_launch(att, e->F, BR, e->F, e->in_att.hi, e->in_att.lo, e->in_att.ld, st)) return 1;
        in.hi = e->in_att.hi; in.lo = e->in_att.lo;
        // the planes have their own pitch: route through an explicit segment below
    }
    {
        GemmProblem g;
        g.M = BR; g.N = D; g.nseg = 1;
        g.seg[0] = seg_of(in, w.att_embed_w, e->F, e->p_att, e->F);
        g.seg[0].lda_h = e->in_att.ld;
        g.epi.bias = w.att_embed_b; g.epi.relu = 1;
        g.epi.C = e->ex.v.f; g.epi.ldc = e->ex.v.ld;
        if (e->gemm(S_ATT, g, capBR, st)) return 1;
    }
    if (mask != nullptr) { e->launches++; if (mask_rows_launch(e->ex.v, B, R, D, mask, R, st)) return 1; }
    for (int l = 0; l < e->NE; ++l) {
        const capb200_tfm_enc_layer& L = w.enc[l];
        e->launches++;
        if (layer_norm_launch(BR, D, e->ex.v.f, e->ex.v.ld, L.ln0_a, L.ln0_b, 1e-6f, e->eln.v, st)) return 1;
        if (linear(e, S_ENC + 4 * l, e->eln.v, BR, D, e->enc_qkv_w[l], e->pe_qkv[l], e->enc_qkv_b[l], 3 * D, e->eqkv.v, false, nullptr, 0, capBR, st)) return 1;
        e->launches++;
        if (enc_self_attention_launch(B, R, e->H, e->dk, e->eqkv.v.f, e->eqkv.v.f + D, e->eqkv.v.f + 2 * D, e->eqkv.v.ld, mask, R, e->eatt.v, st)) return 1;
        ActView xo = e->ex.v; xo.hi = xo.lo = nullptr;
        if (linear(e, S_ENC + 4 * l + 1, e->eatt.v, BR, D, L.self_attn.o_w, e->pe_o[l], L.self_attn.o_b, D, xo, false, e->ex.v.f, e->ex.v.ld, capBR, st)) return 1;
        e->launches++;
        if (layer_norm_launch(BR, D, e->ex.v.f, e->ex.v.ld, L.ln1_a, L.ln1_b, 1e-6f, e->eln.v, st)) return 1;
        if (linear(e, S_ENC + 4 * l + 2, e->eln.v, BR, D, L.w1_w, e->pe_w1[l], L.w1_b, Dff, e->eh.v, true, nullptr, 0, capBR, st)) return 1;
        if (linear(e, S_ENC + 4 * l + 3, e->eh.v, BR, Dff, L.w2_w, e->pe_w2[l], L.w2_b, D, xo, false, e->ex.v.f, e->ex.v.ld, capBR, st)) return 1;
    }
    e->launches++;
    if (layer_norm_launch(BR, D, e->ex.v.f, e->ex.v.ld, w.enc_norm_a, w.enc_norm_b, 1e-6f, e->mem.v, st)) return 1;
    for (int l = 0; l < e->ND; ++l) {
        ActView o; o.f = e->skv[l]; o.ld = 2 * D;
        if (linear(e, S_SKV + l, e->mem.v, BR, D, e->dec_skv_w[l], e->pd_skv[l], e->dec_skv_b[l], 2 * D, o, false, nullptr, 0, capBR, st)) return 1;
    }
    return 0;
}

// one decoder step for `rows` rows at position t
int core_step(capb200_tfm_engine* e, int rows, int rpi, const int* tokens, const int* anc, const long long* labels, long ld_lab, int t, float* logits,
              long ld_logits, int R, const float* mask, cudaStream_t st) {
    const int D = e->D, Dff = e->Dff, capRows = e->capRows;
    const capb200_tfm_weights& w = e->w;
    e->launches++;
    if (embed_pe_launch(rows, D, tokens, w.lut, w.pe + (long)t * D, sqrtf((float)D), e->x.v, st)) return 1;
    ActView xo = e->x.v; xo.hi = xo.lo = nullptr;
    for (int l = 0; l < e->ND; ++l) {
        const capb200_tfm_dec_layer& L = w.dec[l];
        const int s0 = S_DEC + 6 * l;
        e->launches++;
        if (layer_norm_launch(rows, D, e->x.v.f, e->x.v.ld, L.ln0_a, L.ln0_b, 1e-6f, e->ln.v, st)) return 1;
        if (linear(e, s0, e->ln.v, rows, D, e->dec_qkv_w[l], e->pd_qkv[l], e->dec_qkv_b[l], 3 * D, e->qkv.v, false, nullptr, 0, capRows, st)) return 1;
        e->launches++;
        if (dec_self_attention_launch(rows, e->H, e->dk, t, e->qkv.v.f, e->qkv.v.ld, e->kc[l], e->vc[l], e->cache_step_stride, D, anc, e->T, labels,
                                      ld_lab, e->att.v, st)) return 1;
        if (linear(e, s0 + 1, e->att.v, rows, D, L.self_attn.o_w, e->pd_o[l], L.self_attn.o_b, D, xo, false, e->x.v.f, e->x.v.ld, capRows, st)) return 1;
        e->launches++;
        if (layer_norm_launch(rows, D, e->x.v.f, e->x.v.ld, L.ln1_a, L.ln1_b, 1e-6f, e->ln.v, st)) return 1;
        if (linear(e, s0 + 2, e->ln.v, rows, D, L.src_attn.q_w, e->pd_qs[l], L.src_attn.q_b, D, e->qs.v, false, nullptr, 0, capRows, st)) return 1;
        e->launches++;
        if (cross_attention_launch(rows, rpi, e->H, e->dk, R, e->qs.v.f, e->qs.v.ld, e->skv[l], e->skv[l] + D, 2 * D, mask, R, e->att.v, st)) return 1;
        if (linear(e, s0 + 3, e->att.v, rows, D, L.src_attn.o_w, e->pd_os[l], L.src_attn.o_b, D, xo, false, e->x.v.f, e->x.v.ld, capRows, st)) return 1;
        e->launches++;
        if (layer_norm_launch(rows, D, e->x.v.f, e->x.v.ld, L.ln2_a, L.ln2_b, 1e-6f, e->ln.v, st)) return 1;
        if (linear(e, s0 + 4, e->ln.v, rows, D, L.w1_w, e->pd_w1[l], L.w1_b, Dff, e->hh.v, true, nullptr, 0, capRows, st)) return 1;
        if (linear(e, s0 + 5, e->hh.v, rows, Dff, L.w2_w, e->pd_w2[l], L.w2_b, D, xo, false, e->x.v.f, e->x.v.ld, capRows, st)) return 1;
    }
    e->launches++;
    if (layer_norm_launch(rows, D, e->x.v.f, e->x.v.ld, w.dec_norm_a, w.dec_norm_b, 1e-6f, e->ln.v, st)) return 1;
    ActView lo; lo.f = logits; lo.ld = ld_logits;
    return linear(e, S_GEN, e->ln.v, rows, D, w.gen_w, e->p_gen, w.gen_b, e->V1, lo, false, nullptr, 0, capRows, st);
}

}  // namespace

int capb200_tfm_engine::decode_workspace(int B, int rows, int R, int beam, int /*rows_per_image*/, cudaStream_t st) {
    return ensure_workspace(this, B, rows, R, beam, st);
}

int capb200_tfm_engine::decode_prepare(const float* /*fc*/, const float* att, const DecodeCtx& c, cudaStream_t st) {
    return prepare(this, att, c.mask, c.B, c.R, st);
}

// Beam search hands over parent rows from t = 1 on: a beam row then reads its ancestors' cache entries through the search history.  Sampling
// rows read their own; teacher forcing masks the pad keys with the labels.
int capb200_tfm_engine::decode_core(int rows, int rpi, const int* tokens, const int* src_row, int t, float* logits, long ld, const DecodeCtx& c,
                                    cudaStream_t st) {
    const int* anc = (t > 0 && src_row != nullptr) ? beam_ancestors(d.bs, t) : nullptr;
    return core_step(this, rows, rpi, tokens, anc, c.labels, c.ld_labels, t, logits, ld, c.R, c.mask, st);
}

extern "C" {

capb200_tfm_engine* capb200_tfm_create(const capb200_tfm_cfg* c) {
    if (c == nullptr) { set_error("null cfg"); return nullptr; }
    if (c->n_enc < 0 || c->n_enc > CAPB200_TFM_MAX_LAYERS || c->n_dec < 1 || c->n_dec > CAPB200_TFM_MAX_LAYERS) { set_error("layer count must be within 1..8"); return nullptr; }
    if (c->heads < 1 || c->d_model % c->heads != 0) { set_error("d_model must be divisible by the head count"); return nullptr; }
    capb200_tfm_engine* e = create_engine<capb200_tfm_engine>(c->vocab_size, c->seq_length, c->numeric_mode, S_COUNT);
    if (e == nullptr) return nullptr;
    e->cfg = *c;
    e->D = c->d_model; e->Dff = c->d_ff; e->H = c->heads; e->dk = c->d_model / c->heads;
    e->NE = c->n_enc; e->ND = c->n_dec; e->F = c->att_feat_size;
    e->bind_name = "capb200_tfm_bind_weights";
    e->graph_family = 7;
    e->max_teacher_steps = e->T + 1;      // the K/V cache holds bos + T labels
    return e;
}

void capb200_tfm_destroy(capb200_tfm_engine* e) { delete e; }

long capb200_tfm_launch_count(const capb200_tfm_engine* e) { return e ? e->launches : 0; }

int capb200_tfm_bind_weights(capb200_tfm_engine* e, const capb200_tfm_weights* w, void* stream) {
    CAPB_REQUIRE(e != nullptr && w != nullptr, "null argument");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CAPB_REQUIRE(w->att_embed_w && w->att_embed_b && w->lut && w->pe && w->gen_w && w->gen_b && w->dec_norm_a && w->dec_norm_b, "missing weights");
    e->w = *w;
    const int D = e->D, Dff = e->Dff;
    if (e->alloc_wblock(st, [&](Arena& a) { layout_weights(e, a); })) return 1;
    const long dd = (long)D * D;
    for (int l = 0; l < e->NE; ++l) {
        const capb200_mha_weights& a = w->enc[l].self_attn;
        if (concat_rows(e->enc_qkv_w[l], a.q_w, a.k_w, a.v_w, dd, st) || concat_rows(e->enc_qkv_b[l], a.q_b, a.k_b, a.v_b, D, st)) return 1;
    }
    for (int l = 0; l < e->ND; ++l) {
        const capb200_mha_weights& a = w->dec[l].self_attn;
        const capb200_mha_weights& s = w->dec[l].src_attn;
        if (concat_rows(e->dec_qkv_w[l], a.q_w, a.k_w, a.v_w, dd, st) || concat_rows(e->dec_qkv_b[l], a.q_b, a.k_b, a.v_b, D, st)) return 1;
        if (concat_rows(e->dec_skv_w[l], s.k_w, s.v_w, nullptr, dd, st) || concat_rows(e->dec_skv_b[l], s.k_b, s.v_b, nullptr, D, st)) return 1;
    }
    if (e->tc) {
        int rc = pack(e, w->att_embed_w, D, e->F, e->p_att, st) | pack(e, w->gen_w, e->V1, D, e->p_gen, st);
        for (int l = 0; l < e->NE; ++l) {
            rc |= pack(e, e->enc_qkv_w[l], 3 * D, D, e->pe_qkv[l], st) | pack(e, w->enc[l].self_attn.o_w, D, D, e->pe_o[l], st);
            rc |= pack(e, w->enc[l].w1_w, Dff, D, e->pe_w1[l], st) | pack(e, w->enc[l].w2_w, D, Dff, e->pe_w2[l], st);
        }
        for (int l = 0; l < e->ND; ++l) {
            rc |= pack(e, e->dec_qkv_w[l], 3 * D, D, e->pd_qkv[l], st) | pack(e, w->dec[l].self_attn.o_w, D, D, e->pd_o[l], st);
            rc |= pack(e, w->dec[l].src_attn.q_w, D, D, e->pd_qs[l], st) | pack(e, e->dec_skv_w[l], 2 * D, D, e->pd_skv[l], st);
            rc |= pack(e, w->dec[l].src_attn.o_w, D, D, e->pd_os[l], st);
            rc |= pack(e, w->dec[l].w1_w, Dff, D, e->pd_w1[l], st) | pack(e, w->dec[l].w2_w, D, Dff, e->pd_w2[l], st);
        }
        if (rc) return 1;
    }
    return e->finish_bind(st);
}

int capb200_tfm_decode_beam(capb200_tfm_engine* e, const float* att, const float* mask, int B, int R, const capb200_beam_opts* opts, long long* seq,
                            float* seq_logprobs, long long* done_seq, int* done_len, float* done_p, float* done_raw, void* stream) {
    return decode_beam(e, nullptr, att, mask, B, R, opts, seq, seq_logprobs, done_seq, done_len, done_p, done_raw, static_cast<cudaStream_t>(stream));
}

int capb200_tfm_beam_record_logprobs(capb200_tfm_engine* e, int image, int rank, float* dst, void* stream) {
    return decode_record_logprobs(e, image, rank, dst, static_cast<cudaStream_t>(stream));
}

int capb200_tfm_decode_sample(capb200_tfm_engine* e, const float* att, const float* mask, int B, int R, const capb200_sample_opts* opts,
                              const long long* tokens_in, long ld_tok, long long* seq, float* seq_logprobs, float* picked, void* stream) {
    return decode_sample(e, nullptr, att, mask, B, R, opts, tokens_in, ld_tok, seq, seq_logprobs, picked, static_cast<cudaStream_t>(stream));
}

}  // extern "C"


// =====================================================================================================================
// Training steps of the Transformer captioner.
//
// Reference: LossWrapper.forward (captioning/modules/loss_wrapper.py:25-73) over TransformerModel -- the XE branch calls
// TransformerModel._forward (TransformerModel.py:340-348: ONE teacher-forced pass over all positions, seq_mask = pad/eos keys masked +
// subsequent mask, :319-328) and LanguageModelCriterion / LabelSmoothing; the sc branch samples in train mode through core (:351-363,
// which re-runs the whole prefix every step -- causal, so the result equals a K/V-cached step) and applies RewardCriterion; then
// loss.backward() (tools/train.py:189).
//
// Shape of the implementation: decoder activations live on a TIME-major tape (row = t * N + n), so
//   * the teacher-forced pass runs every kernel once over all L * N rows,
//   * the sampling pass runs the same kernels on the N rows of one position per step (the tape's earlier K/V rows are its cache),
//   * the backward pass is always batched over the L * N rows: every contraction is a wgmma tf32 GEMM (gemm_tf32.cu).
// Dropout masks are functions of (seed, site, position, element), so both forward forms draw the same masks.  Sites: 1 att_embed;
// 2 target embedding + positional encoding; encoder layer l: 10+l attention probabilities, 20+l / 40+l the two SublayerConnections,
// 30+l the feed-forward hidden layer; decoder layer l: 50+l self-attention probabilities, 60+l / 80+l / 100+l the three
// SublayerConnections, 70+l source-attention probabilities, 90+l the feed-forward hidden layer.
// One deviation, documented in DESIGN.md: _forward repeats the image features per caption BEFORE the encoder (:329-333), so the
// reference runs the encoder seq_per_img times per image with independent dropout masks; here the encoder runs once per image and its
// output is shared by the image's captions (identical when dropout is off; with dropout on, one encoder mask per image instead of five).
// =====================================================================================================================
namespace {

constexpr int TML = CAPB200_TFM_MAX_LAYERS;

struct TTape : StepTape {
    // encoder, rows b * R + r
    float *X[TML + 1], *eln0[TML], *eqkv[TML], *eatt[TML], *xm[TML], *eln1[TML], *ehd[TML], *mem, *skv[TML];
    // decoder, rows t * N + n
    float *Y[TML + 1], *dln0[TML], *dqkv[TML], *datt[TML], *ym1[TML], *dln1[TML], *dqs[TML], *probs[TML], *dcatt[TML], *ym2[TML], *dln2[TML], *dhd[TML];
    float *yln_tm, *yln_nm;
    int* tok;
    float* key_mask;
    // gradients / scratch
    float *d_yln_nm, *dY, *d_tmp, *d_h, *d_ln, *d_att, *d_qs, *d_qkv, *d_skv[TML], *d_mem, *dX, *tmp, *stats;
};

void layout_ttape(TTape& tp, Arena& a, int B, int R, int N, int T, int D, int Dff, int heads, int V1, int NE, int ND, long glp_floats) {
    const long BR = (long)B * R, TN = (long)T * N;
    const long big = BR > TN ? BR : TN;
    for (int l = 0; l <= NE; ++l) tp.X[l] = a.take<float>(BR * D);
    for (int l = 0; l < NE; ++l) {
        tp.eln0[l] = a.take<float>(BR * D); tp.eqkv[l] = a.take<float>(BR * 3 * D); tp.eatt[l] = a.take<float>(BR * D); tp.xm[l] = a.take<float>(BR * D);
        tp.eln1[l] = a.take<float>(BR * D); tp.ehd[l] = a.take<float>(BR * Dff);
    }
    tp.mem = a.take<float>(BR * D);
    for (int l = 0; l < ND; ++l) { tp.skv[l] = a.take<float>(BR * 2 * D); tp.d_skv[l] = a.take<float>(BR * 2 * D); }
    for (int l = 0; l <= ND; ++l) tp.Y[l] = a.take<float>(TN * D);
    for (int l = 0; l < ND; ++l) {
        tp.dln0[l] = a.take<float>(TN * D); tp.dqkv[l] = a.take<float>(TN * 3 * D); tp.datt[l] = a.take<float>(TN * D); tp.ym1[l] = a.take<float>(TN * D);
        tp.dln1[l] = a.take<float>(TN * D); tp.dqs[l] = a.take<float>(TN * D); tp.probs[l] = a.take<float>(TN * heads * R); tp.dcatt[l] = a.take<float>(TN * D);
        tp.ym2[l] = a.take<float>(TN * D); tp.dln2[l] = a.take<float>(TN * D); tp.dhd[l] = a.take<float>(TN * Dff);
    }
    tp.yln_tm = a.take<float>(TN * D); tp.yln_nm = a.take<float>(TN * D);
    tp.tok = a.take<int>(TN);
    tp.key_mask = a.take<float>(TN);
    tp.layout(a, B, N, TN, V1, glp_floats);
    tp.d_yln_nm = a.take<float>(TN * D); tp.dY = a.take<float>(TN * D);
    tp.d_tmp = a.take<float>(big * D); tp.d_h = a.take<float>(big * Dff); tp.d_ln = a.take<float>(big * D); tp.d_att = a.take<float>(big * D);
    tp.d_qs = a.take<float>(TN * D); tp.d_qkv = a.take<float>(big * 3 * D); tp.d_mem = a.take<float>(BR * D); tp.dX = a.take<float>(BR * D);
    tp.tmp = a.take<float>(big * D);
    tp.stats = a.take<float>(2 * big);
}

// the shared arguments (positions evaluated: XE label_cols - 1, SCST seq_length; p = the Transformer's `dropout`) and att_embed's rate
struct TfmTrainArgs : TrainArgs {
    float p_lm = 0.f;
};

// att_embed's rate (drop_prob_lm of capb200_tfm_xe_opts / capb200_tfm_scst_opts), checked, into `ta`
template <class Opts>
int tfm_rates(const Opts& o, TfmTrainArgs* ta) {
    CAPB_REQUIRE(o.drop_prob_lm >= 0.f && o.drop_prob_lm < 1.f, "dropout rates must be in [0, 1)");
    ta->p_lm = o.drop_prob_lm;
    return 0;
}

// the Transformer's options as the shared option structs (p = its `dropout`); XE evaluates every position (one pass over label_cols - 1
// positions) and has no scheduled sampling
capb200_scst_opts shared_opts(const capb200_tfm_scst_opts& o) {
    return {o.sample_n, o.temperature, o.seed, o.dropout, o.upstream, o.baseline, o.forced_tokens, o.att_masks, o.keep_rows, o.row_loss, o.sampler,
            o.reward_weights};
}
capb200_xe_opts shared_opts(const capb200_tfm_xe_opts& o, int label_cols) {
    return {o.seq_per_img, label_cols - 1, o.seed, o.dropout, o.label_smoothing, o.upstream, o.att_masks, 0.f, nullptr, o.keep_rows, o.row_loss};
}

int tfm_train_step(capb200_tfm_engine* e, const float* att, int B, int R, const TfmTrainArgs& ta, const capb200_tfm_grads* grads, cudaStream_t st) {
    const int n = ta.n, N = B * n, T = ta.T, D = e->D, Dff = e->Dff, V1 = e->V1, F = e->F, heads = e->H, dk = e->dk, NE = e->NE, ND = e->ND;
    const int BR = B * R, TNr = T * N;
    const int idxL = e->T + 2;                         // fixed pitch of the self-attention dropout index (positions never reach it)
    const float p = ta.p, p_lm = ta.p_lm;
    const unsigned long long seed = ta.seed;
    const capb200_tfm_weights& w = e->w;
    const float emb_scale = sqrtf((float)D);
    CAPB_REQUIRE(T >= 1 && T <= e->T + 1, "positions out of range");
    TTape tp;
    if (carve_tape(&e->tape, &e->tape_bytes, tp, st, [&](TTape& tt, Arena& a) {
            layout_ttape(tt, a, B, R, N, T, D, Dff, heads, V1, NE, ND, ta.xe ? 1 : (long)B * e->T * V1);
        })) return 1;

    // ---- greedy baseline (eval mode): the regular K/V-cached decode, forked here, enqueued after the encoder
    if (!ta.xe && ta.greedy_baseline && ensure_workspace(e, B, B, R, 1, st)) return 1;
    StepBaseline gb;
    if (gb.fork(ta, &e->side, &e->ev_fork, &e->ev_join, st)) return 1;
    const Skinny sk = step_gemms(&e->tf32, e->tc, tp, st);
    const long tf32_l0 = tf32_context_launches(e->tf32);
    long& nl = e->launches;
    int rc = 0;

    // ---- encoder forward on the tape (train mode)
    rc |= sk.lin(att, F, w.att_embed_w, F, w.att_embed_b, tp.X[0], D, BR, D, F, 0);
    rc |= relu_dropout_rows_launch(BR, BR, D, 0, tp.X[0], D, seed, 1, p_lm, st);
    if (ta.mask != nullptr) { rc |= mask_rows_launch(f32_view(tp.X[0], D), B, R, D, ta.mask, R, st); nl++; }
    nl += 2;
    for (int l = 0; l < NE && !rc; ++l) {
        const capb200_tfm_enc_layer& Lw = w.enc[l];
        rc |= layer_norm_launch(BR, D, tp.X[l], D, Lw.ln0_a, Lw.ln0_b, 1e-6f, f32_view(tp.eln0[l], D), st);
        rc |= sk.lin(tp.eln0[l], D, e->enc_qkv_w[l], D, e->enc_qkv_b[l], tp.eqkv[l], 3 * D, BR, 3 * D, D, 0);
        rc |= seq_attn_train_launch(B, R, 0, R, heads, dk, 0, R, R, 1, tp.eqkv[l], tp.eqkv[l] + D, tp.eqkv[l] + 2 * D, 3 * D, seed, 10 + l, p, tp.eatt[l], D, ta.mask, R, st);
        rc |= sk.lin(tp.eatt[l], D, Lw.self_attn.o_w, D, Lw.self_attn.o_b, tp.tmp, D, BR, D, D, 0);
        rc |= add_dropout_rows_launch(BR, BR, D, 0, tp.X[l], D, tp.tmp, D, tp.xm[l], D, seed, 20 + l, p, st);
        rc |= layer_norm_launch(BR, D, tp.xm[l], D, Lw.ln1_a, Lw.ln1_b, 1e-6f, f32_view(tp.eln1[l], D), st);
        rc |= sk.lin(tp.eln1[l], D, Lw.w1_w, D, Lw.w1_b, tp.ehd[l], Dff, BR, Dff, D, 0);
        rc |= relu_dropout_rows_launch(BR, BR, Dff, 0, tp.ehd[l], Dff, seed, 30 + l, p, st);
        rc |= sk.lin(tp.ehd[l], Dff, Lw.w2_w, Dff, Lw.w2_b, tp.tmp, D, BR, D, Dff, 0);
        rc |= add_dropout_rows_launch(BR, BR, D, 0, tp.xm[l], D, tp.tmp, D, tp.X[l + 1], D, seed, 40 + l, p, st);
        nl += 10;
    }
    rc |= layer_norm_launch(BR, D, tp.X[NE], D, w.enc_norm_a, w.enc_norm_b, 1e-6f, f32_view(tp.mem, D), st);
    for (int l = 0; l < ND; ++l) rc |= sk.lin(tp.mem, D, e->dec_skv_w[l], D, e->dec_skv_b[l], tp.skv[l], 2 * D, BR, 2 * D, D, 0);
    nl += 1 + ND;
    if (rc) return 1;

    // ---- the greedy baseline's launches are enqueued only now: its stream forked at the top of the step, and while the host enqueues
    // them the main stream is busy with the encoder instead of idle
    if (gb.enqueue(B, e->T, V1, ta.greedy_seq, tp.glp, [&](const capb200_sample_opts* so, const long long* tok, long long* seq, float* lp, void* s) {
            return capb200_tfm_decode_sample(e, att, ta.mask, B, R, so, tok, tok ? e->T : 0, seq, lp, nullptr, s);
        })) return 1;

    // ---- decoder forward over positions [t0, t1)
    const float* key_mask = ta.xe ? tp.key_mask : nullptr;
    auto dec_forward = [&](int t0, int t1) -> int {
        const long r0 = (long)t0 * N;
        const int nr = (t1 - t0) * N;
        int r = 0;
        r |= embed_pe_dropout_launch(nr, N, D, tp.tok + r0, w.lut, w.pe, emb_scale, t0, seed, 2, p, tp.Y[0] + r0 * D, D, st);
        for (int l = 0; l < ND && !r; ++l) {
            const capb200_tfm_dec_layer& Lw = w.dec[l];
            r |= layer_norm_launch(nr, D, tp.Y[l] + r0 * D, D, Lw.ln0_a, Lw.ln0_b, 1e-6f, f32_view(tp.dln0[l] + r0 * D, D), st);
            r |= sk.lin(tp.dln0[l] + r0 * D, D, e->dec_qkv_w[l], D, e->dec_qkv_b[l], tp.dqkv[l] + r0 * 3 * D, 3 * D, nr, 3 * D, D, 0);
            r |= seq_attn_train_launch(N, t1, t0, t1, heads, dk, 1, idxL, 1, N, tp.dqkv[l], tp.dqkv[l] + D, tp.dqkv[l] + 2 * D, 3 * D, seed, 50 + l, p, tp.datt[l], D,
                                       key_mask, T, st);
            r |= sk.lin(tp.datt[l] + r0 * D, D, Lw.self_attn.o_w, D, Lw.self_attn.o_b, tp.tmp, D, nr, D, D, 0);
            r |= add_dropout_rows_launch(nr, N, D, t0, tp.Y[l] + r0 * D, D, tp.tmp, D, tp.ym1[l] + r0 * D, D, seed, 60 + l, p, st);
            r |= layer_norm_launch(nr, D, tp.ym1[l] + r0 * D, D, Lw.ln1_a, Lw.ln1_b, 1e-6f, f32_view(tp.dln1[l] + r0 * D, D), st);
            r |= sk.lin(tp.dln1[l] + r0 * D, D, Lw.src_attn.q_w, D, Lw.src_attn.q_b, tp.dqs[l] + r0 * D, D, nr, D, D, 0);
            r |= cross_attn_train_launch(nr, n, heads, dk, R, tp.dqs[l] + r0 * D, D, tp.skv[l], tp.skv[l] + D, 2 * D, seed, 70 + l, t0, p, tp.dcatt[l] + r0 * D, D,
                                         tp.probs[l] + r0 * heads * R, st, ta.mask, R, N);
            r |= sk.lin(tp.dcatt[l] + r0 * D, D, Lw.src_attn.o_w, D, Lw.src_attn.o_b, tp.tmp, D, nr, D, D, 0);
            r |= add_dropout_rows_launch(nr, N, D, t0, tp.ym1[l] + r0 * D, D, tp.tmp, D, tp.ym2[l] + r0 * D, D, seed, 80 + l, p, st);
            r |= layer_norm_launch(nr, D, tp.ym2[l] + r0 * D, D, Lw.ln2_a, Lw.ln2_b, 1e-6f, f32_view(tp.dln2[l] + r0 * D, D), st);
            r |= sk.lin(tp.dln2[l] + r0 * D, D, Lw.w1_w, D, Lw.w1_b, tp.dhd[l] + r0 * Dff, Dff, nr, Dff, D, 0);
            r |= relu_dropout_rows_launch(nr, N, Dff, t0, tp.dhd[l] + r0 * Dff, Dff, seed, 90 + l, p, st);
            r |= sk.lin(tp.dhd[l] + r0 * Dff, Dff, Lw.w2_w, Dff, Lw.w2_b, tp.tmp, D, nr, D, Dff, 0);
            r |= add_dropout_rows_launch(nr, N, D, t0, tp.ym2[l] + r0 * D, D, tp.tmp, D, tp.Y[l + 1] + r0 * D, D, seed, 100 + l, p, st);
            nl += 16;
        }
        r |= layer_norm_launch(nr, D, tp.Y[ND] + r0 * D, D, w.dec_norm_a, w.dec_norm_b, 1e-6f, f32_view(tp.yln_tm + r0 * D, D), st);
        nl += 2;
        return r;
    };

    const long ld_lp = (long)T * V1;                   // log-prob row pitch of one sequence: [N, T, V1]
    if (ta.xe) {
        if (load_tokens_tm_launch(ta.labels, ta.ld_labels, N, T, tp.tok, tp.key_mask, T, st)) return 1;
        if (dec_forward(0, T)) return 1;
        rc |= permute_rows_launch(T, N, D, tp.yln_tm, D, tp.yln_nm, D, 1, st);
        rc |= sk.lin(tp.yln_nm, D, w.gen_w, D, w.gen_b, ta.logprobs, V1, TNr, V1, D, 0);
        VocabStepArgs va; va.rows = TNr; va.V1 = V1; va.logits = ta.logprobs; va.ld = V1;
        rc |= vocab_step_launch(va, st);
        nl += 4;
        if (rc) return 1;
    } else {
        CAPB_CHECK_CUDA(cudaMemsetAsync(tp.s_tokens, 0, sizeof(int) * N, st));
        for (int t = 0; t < T; ++t) {
            if (feed_tokens(ta, tp, N, V1, t, tp.tok + (long)t * N, st)) return 1;
            if (dec_forward(t, t + 1)) return 1;
            if (sk.lin(tp.yln_tm + (long)t * N * D, D, w.gen_w, D, w.gen_b, ta.logprobs + (long)t * V1, ld_lp, N, V1, D, 0)) return 1;
            if (train_vocab_step(ta, tp, N, V1, t, st)) return 1;
            nl += 3;
        }
        if (permute_rows_launch(T, N, D, tp.yln_tm, D, tp.yln_nm, D, 1, st)) return 1;
        nl += 5;
    }
    if (ta.forward_only) return 0;
    if (loss_backward(ta, tp, gb, B, N, V1, st)) return 1;
    const capb200_tfm_grads& G = *grads;

    // ---- backward: generator and the final LayerNorm
    auto colsum = [&](int rows, int cols, const float* x, long ld, float* out) { nl++; return colsum_launch(rows, cols, x, ld, out, 0, st); };
    rc |= sk.dgrad(TNr, D, V1, tp.DL, V1, w.gen_w, D, tp.d_yln_nm, D, 0);
    rc |= sk.wgrad(V1, D, TNr, tp.DL, V1, tp.yln_nm, D, G.gen_w, D, 0);
    rc |= colsum(TNr, V1, tp.DL, V1, G.gen_b);
    rc |= permute_rows_launch(T, N, D, tp.d_yln_nm, D, tp.d_tmp, D, 0, st);
    rc |= ln_backward_launch(TNr, D, tp.Y[ND], D, w.dec_norm_a, tp.d_tmp, D, 1e-6f, tp.dY, D, 0, tp.stats, G.dec_norm_a, G.dec_norm_b, 0, st);
    nl += 3;
    for (int l = 0; l < ND; ++l) CAPB_CHECK_CUDA(cudaMemsetAsync(tp.d_skv[l], 0, sizeof(float) * (size_t)BR * 2 * D, st));
    if (rc) return 1;
    for (int l = ND - 1; l >= 0 && !rc; --l) {
        const capb200_tfm_dec_layer& Lw = w.dec[l];
        const capb200_tfm_dec_layer_grads& Lg = G.dec[l];
        // feed-forward sublayer: Y[l+1] = ym2 + dropout(w2(dropout(relu(w1(ln2(ym2))))))
        rc |= dropout_rows_copy_launch(TNr, N, D, 0, tp.dY, D, tp.d_tmp, D, seed, 100 + l, p, nullptr, 0, st);
        rc |= sk.wgrad(D, Dff, TNr, tp.d_tmp, D, tp.dhd[l], Dff, Lg.w2_w, Dff, 0);
        rc |= colsum(TNr, D, tp.d_tmp, D, Lg.w2_b);
        rc |= sk.dgrad(TNr, Dff, D, tp.d_tmp, D, Lw.w2_w, Dff, tp.d_h, Dff, 0);
        rc |= dropout_rows_copy_launch(TNr, N, Dff, 0, tp.d_h, Dff, tp.d_h, Dff, seed, 90 + l, p, tp.dhd[l], Dff, st);
        rc |= sk.wgrad(Dff, D, TNr, tp.d_h, Dff, tp.dln2[l], D, Lg.w1_w, D, 0);
        rc |= colsum(TNr, Dff, tp.d_h, Dff, Lg.w1_b);
        rc |= sk.dgrad(TNr, D, Dff, tp.d_h, Dff, Lw.w1_w, D, tp.d_ln, D, 0);
        rc |= ln_backward_launch(TNr, D, tp.ym2[l], D, Lw.ln2_a, tp.d_ln, D, 1e-6f, tp.dY, D, 1, tp.stats, Lg.ln2_a, Lg.ln2_b, 0, st);
        // source attention sublayer: ym2 = ym1 + dropout(o(attention(q(ln1(ym1)), memory)))
        rc |= dropout_rows_copy_launch(TNr, N, D, 0, tp.dY, D, tp.d_tmp, D, seed, 80 + l, p, nullptr, 0, st);
        rc |= sk.wgrad(D, D, TNr, tp.d_tmp, D, tp.dcatt[l], D, Lg.src_attn.o_w, D, 0);
        rc |= colsum(TNr, D, tp.d_tmp, D, Lg.src_attn.o_b);
        rc |= sk.dgrad(TNr, D, D, tp.d_tmp, D, Lw.src_attn.o_w, D, tp.d_att, D, 0);
        rc |= cross_attn_backward_launch(B, n, heads, dk, R, tp.dqs[l], D, tp.skv[l], tp.skv[l] + D, 2 * D, seed, 70 + l, 0, p, tp.probs[l], tp.d_att, D, tp.d_qs, D,
                                         tp.d_skv[l], tp.d_skv[l] + D, 2 * D, st, T, N);
        rc |= sk.wgrad(D, D, TNr, tp.d_qs, D, tp.dln1[l], D, Lg.src_attn.q_w, D, 0);
        rc |= colsum(TNr, D, tp.d_qs, D, Lg.src_attn.q_b);
        rc |= sk.dgrad(TNr, D, D, tp.d_qs, D, Lw.src_attn.q_w, D, tp.d_ln, D, 0);
        rc |= ln_backward_launch(TNr, D, tp.ym1[l], D, Lw.ln1_a, tp.d_ln, D, 1e-6f, tp.dY, D, 1, tp.stats, Lg.ln1_a, Lg.ln1_b, 0, st);
        // self-attention sublayer: ym1 = Y[l] + dropout(o(causal attention(q|k|v(ln0(Y[l])))))
        rc |= dropout_rows_copy_launch(TNr, N, D, 0, tp.dY, D, tp.d_tmp, D, seed, 60 + l, p, nullptr, 0, st);
        rc |= sk.wgrad(D, D, TNr, tp.d_tmp, D, tp.datt[l], D, Lg.self_attn.o_w, D, 0);
        rc |= colsum(TNr, D, tp.d_tmp, D, Lg.self_attn.o_b);
        rc |= sk.dgrad(TNr, D, D, tp.d_tmp, D, Lw.self_attn.o_w, D, tp.d_att, D, 0);
        rc |= seq_attn_backward_launch(N, T, heads, dk, 1, idxL, 1, N, tp.dqkv[l], tp.dqkv[l] + D, tp.dqkv[l] + 2 * D, 3 * D, seed, 50 + l, p, tp.d_att, D, tp.d_qkv,
                                       tp.d_qkv + D, tp.d_qkv + 2 * D, 3 * D, key_mask, T, st);
        rc |= qkv_grads(sk, TNr, D, tp.d_qkv, tp.dln0[l], Lg.self_attn, &nl, st);
        rc |= sk.dgrad(TNr, D, 3 * D, tp.d_qkv, 3 * D, e->dec_qkv_w[l], D, tp.d_ln, D, 0);
        rc |= ln_backward_launch(TNr, D, tp.Y[l], D, Lw.ln0_a, tp.d_ln, D, 1e-6f, tp.dY, D, 1, tp.stats, Lg.ln0_a, Lg.ln0_b, 0, st);
        nl += 14;
    }
    if (rc) return 1;
    CAPB_CHECK_CUDA(cudaMemsetAsync(G.lut, 0, sizeof(float) * (size_t)V1 * D, st));
    rc |= embed_pe_backward_launch(TNr, N, D, tp.tok, emb_scale, 0, seed, 2, p, tp.dY, D, G.lut, st);
    // memory: K | V projections of every decoder layer
    for (int l = 0; l < ND; ++l) {
        const capb200_tfm_dec_layer_grads& Lg = G.dec[l];
        rc |= sk.dgrad(BR, D, 2 * D, tp.d_skv[l], 2 * D, e->dec_skv_w[l], D, tp.d_mem, D, l > 0 ? 1 : 0);
        if (Lg.src_attn.v_w == Lg.src_attn.k_w + (long)D * D) rc |= sk.wgrad(2 * D, D, BR, tp.d_skv[l], 2 * D, tp.mem, D, Lg.src_attn.k_w, D, 0);
        else {
            rc |= sk.wgrad(D, D, BR, tp.d_skv[l], 2 * D, tp.mem, D, Lg.src_attn.k_w, D, 0);
            rc |= sk.wgrad(D, D, BR, tp.d_skv[l] + D, 2 * D, tp.mem, D, Lg.src_attn.v_w, D, 0);
        }
        if (Lg.src_attn.v_b == Lg.src_attn.k_b + D) rc |= colsum(BR, 2 * D, tp.d_skv[l], 2 * D, Lg.src_attn.k_b);
        else {
            rc |= colsum(BR, D, tp.d_skv[l], 2 * D, Lg.src_attn.k_b);
            rc |= colsum(BR, D, tp.d_skv[l] + D, 2 * D, Lg.src_attn.v_b);
        }
    }
    if (rc) return 1;
    if (record_group_event(e->grad_events[0], st)) return 1;                                    // generator + decoder + target embedding
    rc |= ln_backward_launch(BR, D, tp.X[NE], D, w.enc_norm_a, tp.d_mem, D, 1e-6f, tp.dX, D, 0, tp.stats, G.enc_norm_a, G.enc_norm_b, 0, st);
    for (int l = NE - 1; l >= 0 && !rc; --l) {
        const capb200_tfm_enc_layer& Lw = w.enc[l];
        const capb200_tfm_enc_layer_grads& Lg = G.enc[l];
        rc |= dropout_rows_copy_launch(BR, BR, D, 0, tp.dX, D, tp.d_tmp, D, seed, 40 + l, p, nullptr, 0, st);
        rc |= sk.wgrad(D, Dff, BR, tp.d_tmp, D, tp.ehd[l], Dff, Lg.w2_w, Dff, 0);
        rc |= colsum(BR, D, tp.d_tmp, D, Lg.w2_b);
        rc |= sk.dgrad(BR, Dff, D, tp.d_tmp, D, Lw.w2_w, Dff, tp.d_h, Dff, 0);
        rc |= dropout_rows_copy_launch(BR, BR, Dff, 0, tp.d_h, Dff, tp.d_h, Dff, seed, 30 + l, p, tp.ehd[l], Dff, st);
        rc |= sk.wgrad(Dff, D, BR, tp.d_h, Dff, tp.eln1[l], D, Lg.w1_w, D, 0);
        rc |= colsum(BR, Dff, tp.d_h, Dff, Lg.w1_b);
        rc |= sk.dgrad(BR, D, Dff, tp.d_h, Dff, Lw.w1_w, D, tp.d_ln, D, 0);
        rc |= ln_backward_launch(BR, D, tp.xm[l], D, Lw.ln1_a, tp.d_ln, D, 1e-6f, tp.dX, D, 1, tp.stats, Lg.ln1_a, Lg.ln1_b, 0, st);
        rc |= dropout_rows_copy_launch(BR, BR, D, 0, tp.dX, D, tp.d_tmp, D, seed, 20 + l, p, nullptr, 0, st);
        rc |= sk.wgrad(D, D, BR, tp.d_tmp, D, tp.eatt[l], D, Lg.self_attn.o_w, D, 0);
        rc |= colsum(BR, D, tp.d_tmp, D, Lg.self_attn.o_b);
        rc |= sk.dgrad(BR, D, D, tp.d_tmp, D, Lw.self_attn.o_w, D, tp.d_att, D, 0);
        rc |= seq_attn_backward_launch(B, R, heads, dk, 0, R, R, 1, tp.eqkv[l], tp.eqkv[l] + D, tp.eqkv[l] + 2 * D, 3 * D, seed, 10 + l, p, tp.d_att, D, tp.d_qkv,
                                       tp.d_qkv + D, tp.d_qkv + 2 * D, 3 * D, ta.mask, R, st);
        rc |= qkv_grads(sk, BR, D, tp.d_qkv, tp.eln0[l], Lg.self_attn, &nl, st);
        rc |= sk.dgrad(BR, D, 3 * D, tp.d_qkv, 3 * D, e->enc_qkv_w[l], D, tp.d_ln, D, 0);
        rc |= ln_backward_launch(BR, D, tp.X[l], D, Lw.ln0_a, tp.d_ln, D, 1e-6f, tp.dX, D, 1, tp.stats, Lg.ln0_a, Lg.ln0_b, 0, st);
        nl += 8;
    }
    rc |= dropout_rows_copy_launch(BR, BR, D, 0, tp.dX, D, tp.d_tmp, D, seed, 1, p_lm, tp.X[0], D, st);
    rc |= sk.wgrad(D, F, BR, tp.d_tmp, D, att, F, G.att_embed_w, F, 0);
    rc |= colsum(BR, D, tp.d_tmp, D, G.att_embed_b);
    nl += 2 + tf32_context_launches(e->tf32) - tf32_l0;
    if (!rc && record_group_event(e->grad_events[1], st)) return 1;                             // encoder + att_embed
    return rc;
}

}  // namespace

extern "C" int capb200_tfm_set_grad_events(capb200_tfm_engine* e, void* const* events, int n) { return set_grad_events(e, events, n); }

extern "C" int capb200_tfm_xe_step(capb200_tfm_engine* e, const float* att, int B, int R, const capb200_tfm_xe_opts* opts, const long long* labels,
                                   const float* masks, int label_cols, const capb200_tfm_grads* grads, float* logprobs, float* loss, void* stream) {
    if (check_ready(e)) return 1;
    CAPB_REQUIRE(opts && att && labels && masks && grads && logprobs && loss, "null argument");
    CAPB_REQUIRE(R >= 1, "attention features required");
    TfmTrainArgs ta;
    if (tfm_rates(*opts, &ta) || xe_train_args(B, shared_opts(*opts, label_cols), labels, masks, label_cols, logprobs, loss, e->T, &ta)) return 1;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return run_eager_step(st, [&] { return tfm_train_step(e, att, B, R, ta, grads, st); });
}

extern "C" int capb200_tfm_scst_step(capb200_tfm_engine* e, const float* att, int B, int R, const capb200_tfm_scst_opts* opts, const capb200_cider_table* table,
                                     const int* refs, const int* ref_offsets, int L, const capb200_tfm_grads* grads, long long* sample_seq, long long* greedy_seq,
                                     float* sample_logprobs, float* reward, float* loss, void* stream) {
    if (check_ready(e)) return 1;
    CAPB_REQUIRE(opts && att && table && refs && ref_offsets && grads && sample_seq && sample_logprobs && reward && loss, "null argument");
    CAPB_REQUIRE(R >= 1, "attention features required");
    TfmTrainArgs ta;
    if (tfm_rates(*opts, &ta) ||
        scst_train_args(B, shared_opts(*opts), table, refs, ref_offsets, L, sample_seq, greedy_seq, sample_logprobs, reward, loss, e->T, &ta)) return 1;
    return run_scst_step(e, opts, grads, ta, nullptr, 0, att, sizeof(float) * (size_t)B * R * e->F, B, R, static_cast<cudaStream_t>(stream),
                         [&](const float*, const float* att_s, const TfmTrainArgs& t, cudaStream_t s) { return tfm_train_step(e, att_s, B, R, t, grads, s); });
}

// PPO (include/capb200.h: capb200_ppo_opts): the sampled step with the PPO criterion; the old policy's teacher-forced pass runs on `old`.
extern "C" int capb200_tfm_ppo_step(capb200_tfm_engine* e, capb200_tfm_engine* old, const float* att, int B, int R, const capb200_tfm_scst_opts* opts,
                                    const capb200_ppo_opts* ppo, const capb200_cider_table* table, const int* refs, const int* ref_offsets, int L,
                                    const capb200_tfm_grads* grads, long long* sample_seq, float* sample_logprobs, float* scores, float* loss, float* pg_loss,
                                    float* kl_loss, float* clipfrac, void* stream) {
    if (check_ready(e)) return 1;
    CAPB_REQUIRE(opts && att && table && refs && ref_offsets && grads && sample_seq && sample_logprobs && loss, "null argument");
    CAPB_REQUIRE(R >= 1, "attention features required");
    TfmTrainArgs ta;
    if (tfm_rates(*opts, &ta) ||
        scst_train_args(B, shared_opts(*opts), table, refs, ref_offsets, L, sample_seq, nullptr, sample_logprobs, nullptr, loss, e->T, &ta)) return 1;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return run_ppo_step(e, old, ppo, ta, B, scores, pg_loss, kl_loss, clipfrac, st,
                        [&](const capb200_sample_opts* so, const long long* tok, float* lo, void* s) {
                            return capb200_tfm_decode_sample(old, att, ta.mask, B, R, so, tok, e->T, nullptr, lo, nullptr, s);
                        },
                        [&] { return tfm_train_step(e, att, B, R, ta, grads, st); });
}

// The autograd entry points (include/capb200.h: capb200_vjp_opts) on the Transformer's option structs.
extern "C" int capb200_tfm_xe_vjp(capb200_tfm_engine* e, const float* att, int B, int R, const capb200_tfm_xe_opts* opts, const capb200_vjp_opts* vjp,
                                  const long long* labels, int label_cols, const capb200_tfm_grads* grads, float* logprobs, void* stream) {
    if (check_ready(e)) return 1;
    CAPB_REQUIRE(opts && vjp && att && labels && logprobs && (grads || vjp->forward_only), "null argument");
    CAPB_REQUIRE(R >= 1, "attention features required");
    TfmTrainArgs ta;
    if (tfm_rates(*opts, &ta) || xe_train_args(B, shared_opts(*opts, label_cols), labels, nullptr, label_cols, logprobs, nullptr, e->T, &ta, vjp)) return 1;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return run_vjp_step(e, st, [&] { return tfm_train_step(e, att, B, R, ta, grads, st); });
}

extern "C" int capb200_tfm_scst_vjp(capb200_tfm_engine* e, const float* att, int B, int R, const capb200_tfm_scst_opts* opts, const capb200_vjp_opts* vjp,
                                    const capb200_tfm_grads* grads, long long* sample_seq, float* sample_logprobs, void* stream) {
    if (check_ready(e)) return 1;
    CAPB_REQUIRE(opts && vjp && att && sample_seq && sample_logprobs && (grads || vjp->forward_only), "null argument");
    CAPB_REQUIRE(R >= 1, "attention features required");
    capb200_scst_opts shared = shared_opts(*opts);
    shared.reward_weights = nullptr;     // no reward runs under the autograd entry points
    TfmTrainArgs ta;
    if (tfm_rates(*opts, &ta) ||
        scst_train_args(B, shared, nullptr, nullptr, nullptr, 0, sample_seq, nullptr, sample_logprobs, nullptr, nullptr, e->T, &ta, vjp)) return 1;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return run_vjp_step(e, st, [&] { return tfm_train_step(e, att, B, R, ta, grads, st); });
}
