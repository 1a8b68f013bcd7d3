// Internal launch prototypes shared by the kernel translation units and the engine.
#pragma once
#include "common.cuh"

namespace capb200 {

// An activation matrix [rows, cols] kept as fp32 and (tensor-core modes) as split-fp16 planes, common pitch `ld`.
struct ActView {
    float* f = nullptr;
    __half* hi = nullptr;
    __half* lo = nullptr;
    long ld = 0;
};

// One state tensor to reorder by parent row: dst[r, :] = src[src_row[r], :]
struct StateCopy {
    const float* src = nullptr;
    long ld_src = 0;
    ActView dst;
};

// Columns 4*c4 .. 4*c4+3 of row r of one or two states: dst[r] = src[src_row] (zeros for src_row < 0), as fp32 and the split-fp16 planes
// when dst has them.  16-byte aligned rows (H, ld_src and dst.ld multiples of 4).  The loads of both states are issued before any store.
__device__ __forceinline__ void copy_states4(long r, int src, int c4, int nstate, const StateCopy& sc0, const StateCopy& sc1) {
    float4 v0 = make_float4(0.f, 0.f, 0.f, 0.f), v1 = v0;
    if (src >= 0) {
        v0 = *reinterpret_cast<const float4*>(sc0.src + (long)src * sc0.ld_src + 4 * c4);
        if (nstate > 1) v1 = *reinterpret_cast<const float4*>(sc1.src + (long)src * sc1.ld_src + 4 * c4);
    }
    for (int s = 0; s < nstate; ++s) {
        const ActView& o = (s == 0) ? sc0.dst : sc1.dst;
        const float4 v = (s == 0) ? v0 : v1;
        *reinterpret_cast<float4*>(o.f + r * o.ld + 4 * c4) = v;
        if (o.hi != nullptr) {
            __align__(8) __half h[4];
            __align__(8) __half l[4];
            split_f32(v.x, h[0], l[0]); split_f32(v.y, h[1], l[1]); split_f32(v.z, h[2], l[2]); split_f32(v.w, h[3], l[3]);
            *reinterpret_cast<uint2*>(o.hi + r * o.ld + 4 * c4) = *reinterpret_cast<const uint2*>(h);
            *reinterpret_cast<uint2*>(o.lo + r * o.ld + 4 * c4) = *reinterpret_cast<const uint2*>(l);
        }
    }
}

// ---- pointwise.cu
int state_gather_embed_launch(int rows, const int* tokens, const int* src_row, const float* emb, long ld_emb, int E, int relu,
                              ActView xt, int H, int nstate, StateCopy sc0, StateCopy sc1, cudaStream_t stream);
int lstm_pointwise_launch(int rows, int H, const float* gates, long ld_g, const int* src_row, const float* c_prev, long ld_cp,
                          float* c_out, long ld_co, ActView h_out, const float* gather_bias, long ld_gb, const int* gather_idx,
                          cudaStream_t stream);
int relu_copy_launch(const float* x, long n, ActView out_flat, cudaStream_t stream);   // out = relu(x) (+ split planes), flat
int lstm_ln_launch(int rows, int H, const float* gates, long ld_g, const float* c_prev, long ld_cp, float* c_out, long ld_co, float* h_out, long ld_h,
                   const float* ln_a, const float* ln_b, float eps, float* ln_out, long ld_ln, cudaStream_t stream);   // LSTM cell + LayerNorm of h
int maxout_pointwise_launch(int rows, int H, const float* sums, long ld_s, const int* src_row, const float* c_prev, long ld_cp,
                            float* c_out, long ld_co, ActView h_out, cudaStream_t stream);
int additive_attention_launch(int n_images, int rpi, int R, int A, int H, const float* att_h, long ld_ah, const float* p_att, long ld_pa,
                              const float* att, long ld_at, const float* mask, long ld_mask, const float* alpha_w, const float* alpha_b,
                              float* score_scratch /*[rows, R]*/, ActView out, cudaStream_t stream, float* alpha_out = nullptr /*[rows, R]*/);
int mask_rows_launch(ActView x, int n_images, int R, int cols, const float* mask, long ld_mask, cudaStream_t stream);
// scheduled sampling: tok_out[r] = label[r, col] or, with probability prob, a draw from exp(prev_logp[r, :])
int ss_select_launch(int rows, int V1, const float* prev_logp, long ld, const long long* labels, long ld_labels, int col, unsigned long long seed, float prob,
                     int* tok_out, cudaStream_t stream);

// Edits of a log-prob row before the next word is chosen (capb200_decode_edits in include/capb200.h)
struct DecodeEdits {
    int constraint = 0;
    int unk_col = -1;
    int n_bad = 0;
    const int* bad = nullptr;
    int trigrams = 0;
    int trigram_rows = 0;
    __host__ __device__ bool any() const { return constraint != 0 || unk_col >= 0 || n_bad > 0 || trigrams != 0; }
    __host__ __device__ int kinds() const { return (constraint ? 1 : 0) + (unk_col >= 0 ? 1 : 0) + (n_bad > 0 ? 1 : 0); }
};

// ---- vocab.cu : log-softmax over the vocabulary + candidate selection
struct VocabStepArgs {
    int rows = 0;
    int V1 = 0;
    float* logits = nullptr;      // [rows, V1] in/out: overwritten with log-probs (pitch ld)
    long ld = 0;
    int twice = 0;                // beam search renormalises the log-probs a second time (CaptionModel.py:204)
    float2* stats = nullptr;      // beam search: keep the raw logits in place and write (max, log-sum-exp) per row here instead
    // top-k output for beam search (k <= 16)
    int topk = 0;
    float* top_val = nullptr;     // [rows, topk]
    int* top_idx = nullptr;       // [rows, topk]
    // greedy / multinomial selection for _sample
    int select = 0;               // 0 none, 1 greedy argmax, 2 multinomial (Gumbel-max on logp / temperature), 3 forced tokens,
                                  // 4 top-k sampling, 5 nucleus (top-p) sampling
    float top = 0.f;              // k (select 4) or p (select 5)
    DecodeEdits edits;            // applied after the log-softmax, before the selection; the edited row is what is stored
    const int* prev_tokens = nullptr;   // [rows] the word fed into this step (for the edits; only read when t > 0)
    float temperature = 1.0f;
    unsigned long long seed = 0;
    unsigned long long step = 0;  // Philox offset: one independent stream per (row, step)
    const int* forced = nullptr;  // [rows] when select == 3
    int* unfinished = nullptr;    // [rows] in/out (nullptr at beam search); rows already finished emit pad and a zero row
    int first_step = 0;
    int* tokens_out = nullptr;    // [rows] next input token
    long long* seq_out = nullptr; // seq[row * ld_seq + t] = token (int64, reference dtype)
    long ld_seq = 0;
    int t = 0;
    float* picked_lp = nullptr;   // optional: picked_lp[row * ld_picked] = log-prob of the chosen token
    long ld_picked = 1;
    // diverse beam search (image-major rows, `first_beam` rows per image in groups of `first_group_rows`): the rows of group `first_group`
    // are at their group's first step and get a single log_softmax (the shared init_logprobs, AttModel.py:239); off when first_beam == 0
    int first_beam = 0, first_group_rows = 1, first_group = -1;
    __host__ __device__ int row_twice(int r) const {
        return twice && !(first_beam > 0 && (r % first_beam) / first_group_rows == first_group);
    }
};
int vocab_step_launch(const VocabStepArgs& a, cudaStream_t stream);
// beam search with decode edits: the per-row candidate list [rows, k_in] (k_in = beam + edits.kinds()) is edited and cut to [rows, beam];
// first_* as in VocabStepArgs (those rows are edited as at step 0)
int beam_edit_launch(int rows, int k_in, int beam, int t, const DecodeEdits& ed, const int* prev_tokens, const float* val_in, const int* idx_in,
                     float* val_out, int* idx_out, cudaStream_t stream, int first_beam = 0, int first_group_rows = 1, int first_group = -1);
// x[r, :] *= factor; with skip_beam > 0 the rows r with (r % skip_beam) / skip_group_rows == skip_group are left alone (diverse beam search)
int scale_rows_launch(float* x, long ld, int rows, int cols, float factor, cudaStream_t stream, int skip_beam = 0, int skip_group_rows = 1,
                      int skip_group = -1);

// ---- beam.cu
struct BeamState {
    int B = 0, beam = 0, T = 0, V1 = 0;
    float* sums = nullptr;        // [B, beam]
    int* seq_a = nullptr;         // [B, beam, T] ping
    int* seq_b = nullptr;         // [B, beam, T] pong
    int* hist_a = nullptr;        // [B, beam, T] row index into the step-s log-prob slab, ping
    int* hist_b = nullptr;
    int* done_cnt = nullptr;      // [B]
    int* done_seq = nullptr;      // [B, beam*T, T]
    int* done_hist = nullptr;     // [B, beam*T, T]
    int* done_len = nullptr;      // [B, beam*T]
    double* done_p = nullptr;     // [B, beam*T]  length-penalised score (the reference keeps Python floats)
    float* done_raw = nullptr;    // [B, beam*T]  raw sum of log-probs
    int* tokens = nullptr;        // [B*beam] next input tokens
    int* src_row = nullptr;       // [B*beam] parent row (index into the previous step's rows)
};
int beam_step_launch(const BeamState& s, int t, int live, const float* top_val, const int* top_idx, int penalty_kind, float penalty_alpha,
                     cudaStream_t stream);
// The two recurrent states (H columns each) a fused beam step gathers by the chosen parents for the next step: dst[r] = src[s.src_row[r]]
struct NextStateGather {
    StateCopy s0, s1;
    int H = 0;
};
// Step t of the search in one launch per image: the vocabulary statistics / top-k of `a` (stats form, a.topk = s.beam, a.rows = B * live),
// beam_step, and for t < T - 1 the gather of `next`.  beam_search_step_applies: 16-byte aligned logit and state rows.
bool beam_search_step_applies(const VocabStepArgs& a, const NextStateGather& next);
int beam_search_step_launch(const BeamState& s, const VocabStepArgs& a, int t, int live, int penalty_kind, float penalty_alpha,
                            const NextStateGather& next, cudaStream_t stream);
// Diverse beam search, global step t (CaptionModel.py:35-209 with G = group_size groups of bdash = s.beam beams, staggered by one step per group).
// `s` describes B*G virtual images of bdash beams (virtual image i*G + g = group g of image i, rows i*G*bdash + g*bdash + j); every group
// active at t (0 <= t - g < T) takes one step in group order: its candidates [rows, k] (k = G*bdash per row) are lowered by lambda times the
// number of earlier groups' beams of the same image holding that word at position t - g, then merged as in beam_step.  Slab rows are
// recorded as g * rows_total + row (the step-(t - g) slab of group g is slab step t).
int diverse_beam_step_launch(const BeamState& s, int G, int t, int k, const float* top_val, const int* top_idx, float lambda, int rows_total,
                             int penalty_kind, float penalty_alpha, cudaStream_t stream);
// sorts each image's finished beams by score, writes the best `keep` records:
//   out_seq [B*keep, T] int64, out_len/out_p [B*keep], out_hist [B*keep, T] (slab rows, -1 beyond length)
int beam_finalize_launch(const BeamState& s, int keep, long long* out_seq, int* out_len, float* out_p, float* out_raw, int* out_hist,
                         cudaStream_t stream);
// dst[k, s, :] = slab[s][hist[k, s], :] (zeros where hist < 0); slab step stride `step_stride` elements
// `stats` (optional): the slab holds raw logits and stats[s * stats_stride + row] = (max, log-sum-exp); rows are normalised on the fly
// (log_softmax once at s == 0, twice afterwards, exactly as the search scored them).
// `seqs` ([nseq, T] int64, the sequences the rows belong to) + `ed`: re-apply the decode edits the search made to each row (optional)
int gather_logprob_rows_launch(const float* slab, long step_stride, long ld_slab, const int* hist, int nseq, int T, int V1, float* dst,
                               const float2* stats, long stats_stride, cudaStream_t stream, const long long* seqs = nullptr,
                               const DecodeEdits* ed = nullptr);

// ---- transformer.cu
int layer_norm_launch(int rows, int D, const float* x, long ld_x, const float* a, const float* b, float eps, ActView out, cudaStream_t st);
int embed_pe_launch(int rows, int D, const int* tokens, const float* lut, const float* pe_row, float scale, ActView out, cudaStream_t st);
// form (here and in the self / cross attention train launchers below): 0 = the staged kernel when its shared-memory footprint fits in 200 KB,
// else the key-tiled one (attn_tiled.cu); 1 = staged only; 2 = key-tiled only (capb200_mha_* op tests)
int enc_self_attention_launch(int B, int R, int heads, int dk, const float* q, const float* k, const float* v, long ld, const float* mask,
                              long ld_mask, ActView out, cudaStream_t st, int form = 0);
// form 0: one lane per position for t < 32 (dec_self_attention_kernel), the chunked online-softmax kernel past it; 1 / 2 force one of the two
int dec_self_attention_launch(int rows, int heads, int dk, int t, const float* qkv, long ld_qkv, float* kcache, float* vcache, long step_stride,
                              long ld_c, const int* anc, long ld_anc, const long long* labels, long ld_lab, ActView out, cudaStream_t st, int form = 0);
int cross_attention_launch(int rows, int rpi, int heads, int dk, int R, const float* q, long ld_q, const float* kk, const float* vv, long ld_kv,
                           const float* mask, long ld_mask, ActView out, cudaStream_t st);

int glu_launch(int rows, int H, const float* t, long ld_t, const float* residual, long ld_res, ActView out, cudaStream_t st);
int masked_mean_launch(int B, int R, int H, const float* x, long ld_x, const float* mask, long ld_mask, ActView out, cudaStream_t st);

// ---- gemm_generic.cu / scst_kernels.cu (training step)
int gemm_generic_launch(int ta, int tb, int M, int N, int K, const float* A, long lda, const float* B, long ldb, float* C, long ldc, int accumulate,
                        const float* bias, cudaStream_t st);
int gemm_skinny_launch(int M, int N, int nseg, const float* const* A, const long* lda, const float* const* B, const long* ldb, const int* K, const int* tb,
                       float* C, long ldc, const float* bias, const float* row_bias, long ld_rb, int rpg, int accumulate, float* scratch,
                       size_t scratch_floats, int mode, cudaStream_t st);   // mode 0 = fp32 CUDA cores, 1 = 3xTF32 mma.sync
int gemm_wgrad_launch(int M, int N, int K, const float* dY, long ld_dy, const float* X, long ld_x, float* G, long ld_g, int accumulate, int mode,
                      cudaStream_t st);   // G[M,N] (+)= dY[K,M]^T X[K,N]; mode 1 = 3xTF32 tensor cores
int colsum_launch(int rows, int cols, const float* x, long ld, float* out, int accumulate, cudaStream_t st);
// ---- gemm_tf32.cu: wgmma tf32 3-pass GEMM on fp32 operands (in-kernel hi/lo split), split-K over a cluster with a DSMEM reduction
struct Tf32Context;      // per-engine cache of encoded tensor maps and transposed operands
Tf32Context* tf32_context_create();
void tf32_context_destroy(Tf32Context* c);
void tf32_context_new_step(Tf32Context* c);          // weights may have changed: per-step transposes are rebuilt on next use
long tf32_context_launches(const Tf32Context* c);
bool gemm_tf32_supported(int nseg, const float* const* X, const long* ldx, const float* const* W, const long* ldw, const int* K);
int gemm_tf32_launch(Tf32Context* ctx, int M, int N, int nseg, const float* const* X, const long* ldx, const float* const* W, const long* ldw, const int* K,
                     float* C, long ldc, const float* bias, const float* row_bias, long ld_rb, int rpg, int accumulate, cudaStream_t st);
const float* tf32_transposed(Tf32Context* ctx, const float* src, long ld_src, int rows, int cols, bool per_step, long* ld_dst, cudaStream_t st);
int dropout_apply_launch(float* x, int rows, int cols, long ld, unsigned long long seed, unsigned site, unsigned step, float p, cudaStream_t st);
// x[r, c] = relu(x[r, c]) * dropmask(site, step, r*cols + c), in place (the logit head's hidden layers in the training steps)
int relu_dropout_apply_launch(float* x, int rows, int cols, long ld, unsigned long long seed, unsigned site, unsigned step, float p, cudaStream_t st);
int dropout_mask_launch(float* m, long n, unsigned long long seed, unsigned site, unsigned step, float p, cudaStream_t st);
int dropout_copy_launch(const float* x, long ld_x, float* y, long ld_y, int rows, int cols, unsigned long long seed, unsigned site, unsigned step, float p,
                        cudaStream_t st);
int embed_relu_dropout_launch(int rows, int E, const int* tokens, const float* emb, float* xt, unsigned long long seed, unsigned step, float p,
                              cudaStream_t st);
int scst_dlogits_launch(const float* logp, long ld_row, const long long* seq, const float* reward, const float* mask_sum, float upstream, int N, int T, int V1,
                        float* dl, cudaStream_t st, const float* row_coef = nullptr);
// drop_worst on the sampled-loss rows: row_msum / row_coef [N] scratch; loss[0] = mean of the `keep` smallest row losses
int scst_drop_worst_launch(const long long* seq, const float* row_loss, int N, int T, int keep, float upstream, float* row_msum, float* row_coef, float* loss,
                           cudaStream_t st);
int xe_loss_backward_launch(const float* logp, long ld_row, const long long* labels, long ld_l, const float* masks, long ld_m, int N, int steps, int Ls, int V1,
                            float smoothing, float upstream, float* mask_sum, float* item_loss, float* dl, float* loss, cudaStream_t st, int keep = 0,
                            float* row_loss = nullptr, float* row_msum = nullptr, float* row_coef = nullptr);
// PPO (losses.py:267-357).  ppo_shift: the old policy's input words [0, seq[:, :-1]] [N, T].  ppo_loss_backward: from the sampled log-probs lp
// (pitch ld_lp between sequences), the old policy's lo [N, T, V1], the per-row advantage adv [N] and the hypothesis scores [N]: d loss / d logits
// into dl [N, T, V1], scores_out [N] (fp32), the per-row losses row_loss [N] (reduction 'none'), pg_loss / kl_loss / clipfrac, and loss: the
// reduction 'mean' loss, or with keep > 0 the mean of the `keep` smallest row losses (drop_worst), whose rows alone get gradients.
struct PpoScratch {
    float* terms;       // [3, N, T]: masked pg, kl and clip terms
    float* row_msum;    // [N]
    float* row_coef;    // [N]
    float* mask_sum;    // [1]
};
int ppo_shift_launch(const long long* seq, int N, int T, long long* tokens_in, cudaStream_t st);
int ppo_loss_backward_launch(const float* lp, long ld_lp, const float* lo, const long long* seq, const float* adv, const double* scores, int N, int T, int V1,
                             float cliprange, float kl_coef, float upstream, int keep, const PpoScratch& s, float* dl, float* scores_out, float* loss,
                             float* row_loss, float* pg_loss, float* kl_loss, float* clipfrac, cudaStream_t st);
// Backward of log_softmax for an outside gradient g = dL/dlogp over [N, T, V1] rows (pitch ld_row between sequences): dl [N, T, V1] =
// g - exp(logp) * rowsum(g); with seq [N, T] (sampling form) the rows of sequences finished before step t get zero.
int logsoftmax_vjp_launch(const float* logp, const float* g, long ld_row, const long long* seq, int N, int T, int V1, float* dl, cudaStream_t st);
int lstm_cell_backward_launch(int rows, int H, const float* gates, const float* c_prev, const float* c_new, const float* dh, const float* dh_extra,
                              long ld_extra, unsigned drop_site, unsigned drop_step, unsigned long long seed, float p, float* dc_carry, float* dgates,
                              cudaStream_t st);
// Att2in2's maxout cell: dsums [rows, 5H] (i, f, o, a, b) from dh (+ dropout-masked dh_extra of site drop_site) and the carried dc
int maxout_cell_backward_launch(int rows, int H, const float* sums, const float* c_prev, const float* c_new, const float* dh, const float* dh_extra,
                                long ld_extra, unsigned drop_site, unsigned drop_step, unsigned long long seed, float p, float* dc_carry, float* dsums,
                                cudaStream_t st);
int attention_backward_launch(int n_images, int rpi, int R, int A, int H, const float* d_out, const float* alpha, const float* att_h, const float* p_att,
                              const float* att, const float* w, float* d_att_h, float* d_att, float* d_p_att, float* d_w, float* d_b, float* d_alpha_scratch,
                              cudaStream_t st);
int relu_dropout_backward_launch(long n, const float* x, const float* dy, float* dx, float scale, cudaStream_t st);
int embed_backward_launch(int rows, int E, const int* tokens, const float* xt, const float* dxt, long ld_dxt, float scale, float* d_emb, cudaStream_t st);
int embed_scatter_launch(int rows, int E, const int* tokens, const float* dxt, long ld_dxt, float* d_emb, cudaStream_t st);   // ungated (bare nn.Embedding)
int per_image_sum_launch(int steps, int rows, int rpi, int cols, const float* x, float* out, cudaStream_t st);
int add_strided_launch(float* a, const float* b, long ld_b, int rows, int cols, cudaStream_t st);

// ---- aoa_train_kernels.cu (AoANet training step)
int ln_backward_launch(int rows, int D, const float* x, long ld_x, const float* a, const float* dy, long ld_dy, float eps, float* dx, long ld_dx, int accumulate,
                       float* stats, float* da, float* db, int accumulate_params, cudaStream_t st, const float* add1 = nullptr, long ld_a1 = 0,
                       const float* add2 = nullptr, long ld_a2 = 0);
// fused element-wise steps of the AoANet decoder loop (aoa_train_kernels.cu)
int aoa_step_inputs_launch(int rows, int E, int H, int rpi, const int* tok_src, int* tok_dst, const float* emb, float* xt, const float* mean, long ld_mean,
                           const float* out_prev, float* x1c, unsigned long long seed, int step, float p_lm, float p_ctx, cudaStream_t st);
int glu_dropout_launch(int rows, int H, const float* t, long ld_t, float* out, long ld_o, float* outd, long ld_d, unsigned long long seed, int step, float p,
                       cudaStream_t st);
int glu_backward_fused_launch(int rows, int H, const float* t, long ld_t, const float* d_outd, long ld_dd, const float* dctx, float* dt, long ld_dt,
                              unsigned long long seed, int step, float p, cudaStream_t st);
int glu_backward_launch(int rows, int H, const float* t, long ld_t, const float* dy, long ld_dy, float* dt, long ld_dt, cudaStream_t st);
// ---- seed salt (dropout.cuh): effective seed of every dropout / sampling kernel = seed argument XOR salt; uploaded in stream order
int dropout_salt_set_scst(unsigned long long salt, cudaStream_t st);
int dropout_salt_set_aoa(unsigned long long salt, cudaStream_t st);
int dropout_salt_set_tfm(unsigned long long salt, cudaStream_t st);
int dropout_salt_set_vocab(unsigned long long salt, cudaStream_t st);
int dropout_salt_set_attn(unsigned long long salt, cudaStream_t st);
inline int dropout_salt_set_all(unsigned long long salt, cudaStream_t st) {
    return dropout_salt_set_scst(salt, st) | dropout_salt_set_aoa(salt, st) | dropout_salt_set_tfm(salt, st) | dropout_salt_set_vocab(salt, st) |
           dropout_salt_set_attn(salt, st);
}
// ---- tfm_train_kernels.cu: element-wise pieces of the Transformer training steps on TIME-major rows (row = t * rps + n; dropout keyed by (t, n))
int embed_pe_dropout_launch(int rows, int rps, int D, const int* tok, const float* lut, const float* pe, float scale, int t0, unsigned long long seed, int site,
                            float p, float* x, long ld, cudaStream_t st);
int embed_pe_backward_launch(int rows, int rps, int D, const int* tok, float scale, int t0, unsigned long long seed, int site, float p, const float* dx, long ld,
                             float* dlut, cudaStream_t st);
int add_dropout_rows_launch(int rows, int rps, int cols, int t0, const float* a, long ld_a, const float* b, long ld_b, float* out, long ld_o, unsigned long long seed,
                            int site, float p, cudaStream_t st);
int dropout_rows_copy_launch(int rows, int rps, int cols, int t0, const float* src, long ld_s, float* dst, long ld_d, unsigned long long seed, int site, float p,
                             const float* relu_of, long ld_r, cudaStream_t st);
int relu_dropout_rows_launch(int rows, int rps, int cols, int t0, float* h, long ld, unsigned long long seed, int site, float p, cudaStream_t st);
int permute_rows_launch(int L, int N, int D, const float* src, long ld_s, float* dst, long ld_d, int to_seq_major, cudaStream_t st);
int load_tokens_tm_launch(const long long* labels, long ld, int N, int L, int* tok, float* key_mask, long ld_m, cudaStream_t st);
// sequence self-attention with replayable dropout (aoa_train_kernels.cu): row(b, pos) = b * b_stride + pos * p_stride
int seq_attn_train_launch(int seqs, int n_keys, int q_lo, int q_hi, int heads, int dk, int causal, int idx_L, long b_stride, long p_stride, const float* q,
                          const float* k, const float* v, long ld, unsigned long long seed, int site, float p, float* out, long ld_out, const float* key_mask,
                          long ld_mask, cudaStream_t st, int form = 0);
int seq_attn_backward_launch(int seqs, int n_keys, int heads, int dk, int causal, int idx_L, long b_stride, long p_stride, const float* q, const float* k,
                             const float* v, long ld, unsigned long long seed, int site, float p, const float* d_out, long ld_do, float* dq, float* dk_,
                             float* dv, long ld_d, const float* key_mask, long ld_mask, cudaStream_t st, int form = 0);
int enc_attn_train_launch(int B, int R, int heads, int dk, const float* q, const float* k, const float* v, long ld, unsigned long long seed, int site, float p,
                          float* out, long ld_out, cudaStream_t st, const float* mask = nullptr, long ld_mask = 0);
int enc_attn_backward_launch(int B, int R, int heads, int dk, const float* q, const float* k, const float* v, long ld, unsigned long long seed, int site, float p,
                             const float* d_out, long ld_do, float* dq, float* dk_, float* dv, long ld_d, cudaStream_t st, const float* mask = nullptr,
                             long ld_mask = 0);
int cross_attn_train_launch(int rows, int rpi, int heads, int dk, int R, const float* q, long ld_q, const float* kk, const float* vv, long ld_kv,
                            unsigned long long seed, int site, int step, float p, float* out, long ld_out, float* probs, cudaStream_t st,
                            const float* mask = nullptr, long ld_mask = 0, int row_mod = 0);
int cross_attn_backward_launch(int B, int rpi, int heads, int dk, int R, const float* q, long ld_q, const float* kk, const float* vv, long ld_kv,
                               unsigned long long seed, int site, int step, float p, const float* probs, const float* d_out, long ld_do, float* dq, long ld_dq,
                               float* dkk, float* dvv, long ld_dkv, cudaStream_t st, int n_steps = 1, int row_mod = 0, int form = 0);
// ---- attn_tiled.cu: key-tiled forms of the above (self-attention, causal or not; cross-attention backward), no footprint grows with the keys.
// causal forward: queries [q_lo, q_hi) (q_hi < 0: n_keys); without causal every query runs against every key
int attn_tiled_forward_launch(int seqs, int n_keys, int heads, int dk, int idx_L, long b_stride, long p_stride, const float* q, const float* k, const float* v,
                              long ld, const float* key_mask, long ld_mask, unsigned long long seed, int site, float p, ActView out, cudaStream_t st,
                              int causal = 0, int q_lo = 0, int q_hi = -1);
int attn_tiled_self_backward_launch(int seqs, int n_keys, int heads, int dk, int idx_L, long b_stride, long p_stride, const float* q, const float* k,
                                    const float* v, long ld, unsigned long long seed, int site, float p, const float* d_out, long ld_do, float* dq, float* dk_,
                                    float* dv, long ld_d, const float* key_mask, long ld_mask, cudaStream_t st, int causal = 0);
int attn_tiled_cross_backward_launch(int B, int rpi1, int n_steps, int row_mod, int heads, int dk, int R, const float* q, long ld_q, const float* kk,
                                     const float* vv, long ld_kv, unsigned long long seed, int site, int step, float p, const float* probs, const float* d_out,
                                     long ld_do, float* dq, long ld_dq, float* dkk, float* dvv, long ld_dkv, cudaStream_t st);
int mean_backward_launch(int B, int R, int H, const float* d_mean, long ld_dm, float* dx, long ld_dx, cudaStream_t st, const float* mask = nullptr,
                         long ld_mask = 0);
int add_dropout_launch(int rows, int cols, const float* a, long ld_a, const float* b, long ld_b, float* out, long ld_o, unsigned long long seed, int site, int step,
                       float p, cudaStream_t st);
int cat_dropout_launch(int rows, int c1, int c2, const float* a, long ld_a, const float* b, long ld_b, float* out, long ld_o, unsigned long long seed, int site,
                       int step, float p, cudaStream_t st);

// ---- reward.cu (CIDEr-D) and criterion
struct CiderTable;   // device hash table of n-gram -> idf
CiderTable* cider_table_create(const int* keys, const double* df, long n, double ref_len, cudaStream_t stream);
void cider_table_destroy(CiderTable* t);
// corpus document frequencies (CiderD(df='corpus')): rebuilt on the device by every reward launch below from its own references
CiderTable* cider_corpus_table_create();
int cider_corpus_table_reserve(CiderTable* t, long n_refs, int L);
bool cider_table_is_corpus(const CiderTable* t);
int corpus_build_launches(const CiderTable* t);       // kernels a reward launch adds to build the table (3 for a corpus table, else 0)
void cider_table_key(const CiderTable* t, unsigned long long key[3]);   // what a captured reward reads: slots, capacity - 1, table kind
int cider_reward_launch(const CiderTable* t, const long long* sampled, int S, const long long* greedy, int B, int T, const int* refs,
                        const int* ref_offsets, int L, double* scores, float* reward, long ld_reward, int reward_cols, cudaStream_t stream);
// per-hypothesis BLEU-4 (float64), hypotheses and references laid out as for cider_reward_launch
int bleu_scores_launch(const long long* sampled, int S, const long long* greedy, int B, int T, const int* refs, const int* ref_offsets, int L,
                       double* scores, cudaStream_t stream);
// scores = w_cider * CIDEr-D + w_bleu * BLEU-4 (a term only when its weight is > 0; t may be null when w_cider <= 0, bleu [hyps] scratch may be null
// when w_bleu <= 0), then the reward as cider_reward_launch writes it
int weighted_reward_launch(const CiderTable* t, double w_cider, double w_bleu, const long long* sampled, int S, const long long* greedy, int B, int T,
                           const int* refs, const int* ref_offsets, int L, double* scores, double* bleu, float* reward, long ld_reward, int reward_cols,
                           cudaStream_t stream);
int weighted_reward_launches(double w_cider, double w_bleu, bool with_reward);     // kernels weighted_reward_launch issues
// coco-caption's Cider() [S] and the per-caption Bleu(4) statistics [S, 6] (correct 1..4-grams, length, closest reference length) over the
// words before each first 0; S / n_images captions per image, each image counted once in the document frequencies of the corpus table t
int coco_cider_bleu_launch(const CiderTable* t, const long long* seqs, int S, int n_images, int T, const int* refs, const int* ref_offsets, int L,
                           double* cider, int* bleu_stats, cudaStream_t stream);

// ---- diversity.cu
// corpus BLEU-1..4 of each round j < n (caption j of every image) from per-caption statistics [n_images, n, 6]: out_bleu[n, 4]
int corpus_bleu_launch(const int* stats, int n_images, int n, double* out_bleu, cudaStream_t stream);
int reward_criterion_fwd_launch(const float* logprobs, long ld_row, long ld_t, const long long* seq, const float* reward, int N, int T,
                                float* loss_mean, float* loss_rows, float* mask_sum, cudaStream_t stream);
int reward_criterion_bwd_launch(const long long* seq, const float* reward, int N, int T, const float* mask_sum, float upstream,
                                float* grad, long ld_row, long ld_t, cudaStream_t stream);

}  // namespace capb200
