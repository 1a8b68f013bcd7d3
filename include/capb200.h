/* capb200 -- C ABI of the H100 (sm_90a) caption-decoding / SCST engine.
 *
 * Drop-in boundary.  The reference (ruotianluo/ImageCaptioning.pytorch) is pure Python and has no FFI layer; its boundary
 * for this path is two Python call surfaces (SURVEY.md section 8b):
 *     CaptionModel.forward(..., mode='sample'|'forward')            captioning/models/CaptionModel.py:29-33
 *       -> AttModel._sample / _sample_beam / _forward              captioning/models/AttModel.py:258,218,126
 *     LossWrapper.forward(..., sc_flag=True)                        captioning/modules/loss_wrapper.py:56-73
 * The Python adapter in imagecaptioning.pytorch_b200 keeps those signatures and calls the entry points below through
 * ctypes.  Every entry point takes plain device pointers and sizes (no torch types), an explicit cudaStream_t passed as
 * void*, is asynchronous with respect to the host unless stated, returns 0 on success and non-zero on failure with a
 * message available from capb200_last_error().  PyTorch owns all tensors; the engine owns only packed weight copies and
 * workspaces.  One engine per device; different engines may be driven from different host threads.
 *
 * All matrices are row-major fp32 unless noted; token ids are int64 (the reference's torch.long) at the boundary.
 */
#ifndef CAPB200_H_
#define CAPB200_H_

#ifdef __cplusplus
extern "C" {
#endif

#define CAPB200_ABI_VERSION 1

/* numeric modes of the dense contractions */
#define CAPB200_MODE_SIMT_FP32 0 /* fp32 FFMA on CUDA cores */
#define CAPB200_MODE_TC_F16X3 1  /* wgmma f16, split-fp16 operands, 3 MMA passes, fp32 accumulate (parity grade) */
#define CAPB200_MODE_TC_F16X1 2  /* wgmma f16, single pass (throughput mode, not parity grade) */
#define CAPB200_MODE_SKINNY_TF32X3 3 /* capb200_linear only: the training step's split-K GEMM, 3xTF32 mma.sync on the fp32 weights */
#define CAPB200_MODE_SKINNY_FP32 4   /* capb200_linear only: same split-K GEMM on CUDA cores */
#define CAPB200_MODE_TF32X3_TC 5       /* capb200_linear only: the training steps' wgmma tf32 3-pass GEMM on fp32 operands (gemm_tf32.cu) */
#define CAPB200_MODE_TF32X3_TC_DGRAD 6 /* same kernel, input-gradient form: y[M,N] = x[M,K] * w[K,N]  (w row-major [K,N], transposed internally) */
#define CAPB200_MODE_TF32X3_TC_WGRAD 7 /* same kernel, weight-gradient form: y[M,N] = x[K,M]^T * w[K,N] (both row-major, transposed internally) */

/* Longest caption every family decodes and trains (seq_length), and the widest hypothesis / reference row the CIDEr-D and BLEU-4
 * rewards score (T and L of the reward entry points, including the closing 0).  256 is what the long BLEU-4 kernel holds: one thread per
 * n-gram (4 orders x 256 positions = 1024 threads, the CTA limit).  Up to 64 tokens the rewards run their original kernels, and up to 31
 * positions the Transformer runs its original decoder self-attention; longer shapes dispatch to the long forms (DESIGN.md, "Caption
 * length").  The diversity entry points (capb200_self_cider, capb200_div_stats) stay at 64 tokens. */
#define CAPB200_MAX_SEQ_LENGTH 256

#define CAPB200_FAMILY_UPDOWN 0 /* UpDownModel  captioning/models/AttModel.py:868 */
#define CAPB200_FAMILY_NEWFC 1  /* NewFCModel   captioning/models/AttModel.py:904 */
#define CAPB200_FAMILY_ATT2IN2 2 /* Att2in2Model captioning/models/AttModel.py:854 (no fc_embed; the core attends with the previous h) */

typedef struct capb200_engine capb200_engine;
typedef struct capb200_cider_table capb200_cider_table;

const char* capb200_last_error(void);
int capb200_abi_version(void);
/* Numeric precondition of the tensor-core modes: every value that is converted to split-fp16 planes (weights at bind time, the fc / att
 * feature tiles of each call) must be finite with |x| < 65504.  A violation sets a process-wide flag; bind_weights checks it synchronously,
 * every later entry point fails with a message while it is set.  Returns the flag (valid once the stream of the offending call has been
 * synchronised); reset != 0 clears it. */
int capb200_range_status(int reset);

/* ------------------------------------------------------------------------------------------------------------------
 * Operator level (each replaces one library call of the reference's per-timestep core; used by the parity tests)
 * ---------------------------------------------------------------------------------------------------------------- */

/* y[M,N] = x[M,K] * w[N,K]^T + b[N] (optional ReLU)             nn.Linear call sites AttModel.py:74-95,172,733
 * mode selects the arithmetic; the tensor-core modes split x and w into fp16 planes in scratch memory first. */
int capb200_linear(const float* x, long ldx, const float* w, long ldw, const float* b, float* y, long ldy, int M, int N, int K,
                   int relu, int mode, void* stream);

/* Same contraction with the operands split once, then `iters` back-to-back launches timed with CUDA events on `stream`
 * (synchronous; y holds the result afterwards).  Used by bench.py / the tiling sweeps. */
int capb200_bench_linear(const float* x, const float* w, const float* b, float* y, int M, int N, int K, int mode, int iters, float* ms_per_launch,
                         void* stream);

/* Diagnostics: the output-tile width (64, 128 or 160 columns) the tc_f16x3 / tc_f16x1 GEMM picks for an M x N problem on the current device. */
int capb200_gemm_tile_n(int M, int N);
/* The output-tile height (128 or 256 rows) the same GEMM picks for an M x N problem; CAPB200_GEMM_BM=128 or 256 in the environment forces
 * it where the tile width has a kernel of that height. */
int capb200_gemm_tile_m(int M, int N);

/* nn.LSTMCell: gates = x*w_ih^T + b_ih + h*w_hh^T + b_hh; (i,f,g,o)           AttModel.py:628,635
 * x[M,Kx], h/c[M,H] -> h_out/c_out[M,H] */
int capb200_lstm_cell(const float* x, int Kx, const float* h, const float* c, const float* w_ih, const float* w_hh, const float* b_ih,
                      const float* b_hh, float* h_out, float* c_out, int M, int H, int mode, void* stream);

/* Attention.forward (AttModel.py:728-748) with per-image features: row r uses image r / rows_per_image.
 * att_h[rows,A] = h2att(h) incl. bias; p_att[B,R,A]; att[B,R,H]; mask[B,R] or NULL; alpha_w[A], alpha_b[1] -> out[rows,H] */
int capb200_additive_attention(const float* att_h, const float* p_att, const float* att, const float* mask, const float* alpha_w,
                               const float* alpha_b, float* out, int n_images, int rows_per_image, int R, int A, int H, void* stream);

/* In-place log_softmax over each row of logits[rows,V1] (twice != 0 applies it a second time, CaptionModel.py:204) and
 * the per-row top-k (values and indices, descending, lowest index first on ties). top_val/top_idx may be NULL if k == 0. */
int capb200_log_softmax_topk(float* logits, long ld, int rows, int V1, int twice, int k, float* top_val, int* top_idx, void* stream);

/* Beam search's form of the same step: logits[rows,V1] (pitch ld) are only read; stats[rows,2] receives each row's maximum and
 * log(sum(exp(x - max))), top_val/top_idx[rows,k] the k best log-probs (normalised a second time if twice != 0) and their columns,
 * ranked on the raw logits (descending, lowest index first on ties), 1 <= k <= 16.  A row with fewer than k entries above -inf
 * fills the rest with value -inf and index 0x7fffffff or a column that holds -inf. */
int capb200_vocab_stats_topk(const float* logits, long ld, int rows, int V1, int twice, int k, float* stats, float* top_val, int* top_idx,
                             void* stream);

/* The word choice of _sample (CaptionModel.py:366-406) on one step's logits[rows,V1] (pitch ld), which are overwritten with their
 * log_softmax.  select: 1 greedy, 2 multinomial, 4 top-k (top = k), 5 nucleus (top = p); the sampled kinds draw from
 * softmax(log-probs / temperature) over the kept words with one Philox block per (word, row, step, seed).  tokens_out[rows] gets the
 * word, picked_lp[rows] its log-prob.  unfinished[rows] (or NULL): unless first_step != 0, a row whose flag is 0 emits word 0, log-prob 0
 * and an all-zero row; the flag is rewritten to word != 0.
 * Supported row lengths: 1 <= V1 <= 409600.  Up to 51200 one CTA holds a row; longer rows are spread over a thread-block cluster of
 * ceil(V1 / 51200) CTAs with the same results (same tie order, same draw for the same seed and step).  V1 > 409600 returns nonzero with
 * the limit in capb200_last_error() before anything is launched (capb200_log_softmax_topk and every sampling / training entry point
 * likewise; capb200_vocab_stats_topk and beam search have no length limit). */
int capb200_vocab_select(float* logits, long ld, int rows, int V1, int select, float top, float temperature, unsigned long long seed,
                         unsigned long long step, int* unfinished, int first_step, int* tokens_out, float* picked_lp, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Engine level
 * ---------------------------------------------------------------------------------------------------------------- */
typedef struct {
    int family;              /* CAPB200_FAMILY_* */
    int vocab_size;          /* V; logits have V+1 entries, id 0 = BOS = EOS = PAD (AttModel.py:65-67) */
    int input_encoding_size; /* E */
    int rnn_size;            /* H */
    int att_hid_size;        /* A */
    int fc_feat_size;        /* F_fc */
    int att_feat_size;       /* F_att */
    int seq_length;          /* T = max_length (AttModel.py:60), 1..CAPB200_MAX_SEQ_LENGTH */
    int numeric_mode;        /* CAPB200_MODE_* */
} capb200_model_cfg;

/* Borrowed fp32 device pointers in the reference's state_dict layouts (SURVEY.md section 8b key list).
 * Att2in2 uses embed, att_embed_*, ctx2att_*, logit_*, h2att_* / alpha_* (core.attention), i2h_* / h2h_* (core.i2h / core.h2h, [5H,E] [5H,H])
 * and a2c_*; its fc_embed_* stay NULL (the model has no fc_embed, AttModel.py:858) and the core never reads the fc features. */
typedef struct {
    const float* embed;                                                           /* [V+1,E]  embed.0.weight | embed.weight */
    const float *fc_embed_w, *fc_embed_b;                                         /* [H,F_fc] (newfc: [E,F_fc]) */
    const float *att_embed_w, *att_embed_b;                                       /* [H,F_att] */
    const float *ctx2att_w, *ctx2att_b;                                           /* [A,H] */
    const float *logit_w, *logit_b;                                               /* [V+1,H] */
    const float *att_lstm_w_ih, *att_lstm_w_hh, *att_lstm_b_ih, *att_lstm_b_hh;   /* [4H,E+2H] [4H,H] [4H] [4H] */
    const float *lang_lstm_w_ih, *lang_lstm_w_hh, *lang_lstm_b_ih, *lang_lstm_b_hh; /* [4H,2H] [4H,H] [4H] [4H] */
    const float *h2att_w, *h2att_b;                                               /* [A,H] */
    const float *alpha_w, *alpha_b;                                               /* [1,A] [1] */
    const float *i2h_w, *i2h_b, *h2h_w, *h2h_b;                                   /* newfc _core: [5H,E] [5H] [5H,H] [5H] */
    const float *a2c_w, *a2c_b;                                                   /* att2in2 core.a2c: [2H,H] [2H] */
} capb200_weights;

capb200_engine* capb200_engine_create(const capb200_model_cfg* cfg);
void capb200_engine_destroy(capb200_engine* e);
/* (Re)binds the parameter tensors; call again after every optimizer step.  Tensor-core modes repack the fp16 planes here. */
int capb200_engine_bind_weights(capb200_engine* e, const capb200_weights* w, void* stream);

/* AttModel's output head for logit_layers = k > 1 (AttModel.py:87-92): the state_dict's logit.0, logit.3, ..., logit.{3(k-2)} are k - 1
 * hidden Linear(H, H) + ReLU + Dropout(0.5) layers ahead of logit.{3(k-1)}, the vocabulary projection (capb200_weights.logit_w / logit_b).
 * The head sits outside the recurrence: the state fed to the next step is the core's output (AttModel.py:166-176).  Every decode (greedy,
 * sampling, teacher forcing, beam and diverse beam search, ensemble members, PPO's old policy) runs the hidden layers before the vocabulary
 * GEMM without dropout (eval mode).  Every training entry point (the fused XE / SCST / PPO steps and the *_vjp autograd entry points) runs
 * them too: hidden layer i's dropout mask at position t is site 200 + i, step t of capb200_dropout_mask under the step's seed, with the rate
 * of set_logit_dropout, and the head's backward runs batched over all positions ahead of backpropagation through time, in gradient group 0.
 * set_logit_layers: k >= 1, once, before the first decode (k = 1, the default, runs exactly the single Linear).
 * bind_logit_head: w[i] [H, H] and b[i] [H] of hidden layer i < k - 1 (logit.{3i}.weight / .bias, fp32, device); call it after every
 * bind_weights (tensor-core modes repack the fp16 planes here).  A decode of an engine with k > 1 and no bound head is refused.
 * bind_logit_head_grads: gw[i] [H, H] and gb[i] [H], OVERWRITTEN by every training call that follows; a training call of an engine with
 * k > 1 and no bound gradient buffers is refused.
 * set_logit_dropout: the hidden layers' dropout rate p in [0, 1) of the training calls that follow: 0.5 (the default; Dropout(0.5) in
 * train mode), 0 for an eval-mode autograd pass. */
int capb200_engine_set_logit_layers(capb200_engine* e, int logit_layers);
int capb200_engine_bind_logit_head(capb200_engine* e, const float* const* w, const float* const* b, void* stream);
int capb200_engine_bind_logit_head_grads(capb200_engine* e, float* const* gw, float* const* gb);
int capb200_engine_set_logit_dropout(capb200_engine* e, float p);

/* Per-step edits of the log-prob rows before the next word is chosen (the reference's decode options; the edited row is also what the
 * reference stores in seqLogprobs / done_beams[...]['logps'], and so do we).  All zero / -1 / NULL = none. */
typedef struct {
    int decoding_constraint;   /* t > 0: log-prob of the previous word = -inf (CaptionModel.py:154-155, AttModel.py:294-297) */
    int unk_col;               /* beam search: this column's log-prob is lowered by 1000 at every step (suppress_UNK with 'UNK' as the last
                                  word, or unk_idx: CaptionModel.py:159-162); -1 = none */
    int n_bad_endings;         /* remove_bad_endings: t > 0 and previous word in the list -> log-prob of the end token (column 0) = -inf
                                  (CaptionModel.py:156-157, AttModel.py:299-304) */
    const int* bad_endings;    /* device, n_bad_endings word ids (model.bad_endings_ix) */
    int block_trigrams;        /* _sample only, t >= 3: every earlier occurrence of (w[t-2], w[t-1], x) lowers x by 2 ln 2 (AttModel.py:306-332) */
    int trigram_rows;          /* rows 0 .. trigram_rows-1 get it (the reference loops over batch_size rows, also when sample_n > 1) */
} capb200_decode_edits;

typedef struct {
    int beam_size;      /* b, 1..16 (with edits: b + number of active edit kinds <= 16) */
    int sample_n;       /* 1 or beam_size (AttModel.py:223) */
    int penalty_kind;   /* 0 '' (identity), 1 'wu_<alpha>', 2 'avg_<alpha>'   captioning/utils/misc.py:133-151 */
    float penalty_alpha;
    float temperature;  /* log_softmax(logprobs / temperature) from the second step on (CaptionModel.py:204); 0 is read as 1 */
    capb200_decode_edits edits;
} capb200_beam_opts;

/* AttModel._sample_beam + CaptionModel.beam_search (group_size 1).
 * fc[B,F_fc], att[B,R,F_att] contiguous, mask[B,R] or NULL.
 * seq[B*sample_n,T] int64 zero padded; seq_logprobs[B*sample_n,T,V+1] (NULL to skip the gather);
 * done_seq[B,b,T] int64, done_len[B,b], done_p[B,b], done_raw[B,b]: each image's finished beams sorted by score (may be NULL). */
int capb200_decode_beam(capb200_engine* e, const float* fc, const float* att, const float* mask, int B, int R, const capb200_beam_opts* opts,
                        long long* seq, float* seq_logprobs, long long* done_seq, int* done_len, float* done_p, float* done_raw, void* stream);
/* capb200_decode_beam with the form of the search step chosen, for tests.  form 0 picks as capb200_decode_beam does: UpDown decodes
 * without edits, at temperature 1 and with 16-byte aligned rows run each step's vocabulary statistics / top-k, beam step and the next
 * step's state gather as one kernel per image.  1 always runs the separate kernels; 2 requires the fused kernel and fails where it does
 * not apply.  Both forms give the same bits. */
int capb200_decode_beam_form(int form, capb200_engine* e, const float* fc, const float* att, const float* mask, int B, int R,
                             const capb200_beam_opts* opts, long long* seq, float* seq_logprobs, long long* done_seq, int* done_len, float* done_p,
                             float* done_raw, void* stream);
/* Full log-prob rows [len, V+1] of finished beam `rank` of image `image` from the most recent capb200_decode_beam call
 * (done_beams[image][rank]['logps'], CaptionModel.py:192); dst must hold T*(V+1) floats, rows beyond the length are zeroed. */
int capb200_beam_record_logprobs(capb200_engine* e, int image, int rank, float* dst, void* stream);

typedef struct {
    capb200_beam_opts base;   /* beam_size = group_size * bdash (bdash beams per group); sample_n 1 or bdash (AttModel.py:223) */
    int group_size;           /* G >= 2, dividing beam_size */
    float diversity_lambda;   /* >= 0: a candidate word loses lambda for every beam of an earlier group holding it at the same position */
} capb200_diverse_opts;

/* Diverse beam search: AttModel._sample_beam + CaptionModel.beam_search with group_size > 1 (CaptionModel.py:35-209), UpDown and Att2in2.
 * Same output contract as capb200_decode_beam, except:
 *   done_*[B, beam]: for each group in order, its bdash best finished beams by score (the reference's group-concatenated done_beams);
 *   seq / seq_logprobs rows k < B: done_beams[k][0] (group 0's best); with sample_n == bdash the rows B .. B*sample_n-1 are pad / zero
 *   (AttModel.py:241-254 fills every sample_n row only when sample_n == beam_size).
 * capb200_beam_record_logprobs reads the records of the last call (rank in 0..beam-1, group order). */
int capb200_decode_beam_diverse(capb200_engine* e, const float* fc, const float* att, const float* mask, int B, int R, const capb200_diverse_opts* opts,
                                long long* seq, float* seq_logprobs, long long* done_seq, int* done_len, float* done_p, float* done_raw, void* stream);

#define CAPB200_SAMPLE_GREEDY 0
#define CAPB200_SAMPLE_MULTINOMIAL 1
#define CAPB200_SAMPLE_FORCED 2  /* replay given tokens (parity checks against another sampler's draw) */
#define CAPB200_SAMPLE_TEACHER 3 /* AttModel._forward: feed labels[:, t] at step t, no finished-row masking */
#define CAPB200_SAMPLE_TOPK 4    /* sample_method 'top<k>', k >= 1: multinomial over the k most likely words of logprobs / temperature
                                    (CaptionModel.py:398-402); `top` = k */
#define CAPB200_SAMPLE_TOPP 5    /* sample_method 'top<p>', 0 < p < 1: nucleus sampling (CaptionModel.py:388-397); `top` = p */
typedef struct {
    int sample_n;             /* rows per image */
    int method;               /* CAPB200_SAMPLE_* */
    float temperature;
    unsigned long long seed;  /* Philox key for the sampling methods */
    int steps;                /* TEACHER: number of label columns to run (<= the label width) */
    float top;                /* TOPK: k, TOPP: p */
    capb200_decode_edits edits;
} capb200_sample_opts;

/* AttModel._sample (greedy / multinomial) and AttModel._forward (teacher forcing).
 * tokens_in[N,ld_tok] int64: forced tokens (FORCED) or labels (TEACHER), else NULL.  N = B*sample_n.
 * seq[N,T] int64; seq_logprobs[N,T_out,V+1] where T_out = T (sampling) or ld_tok (TEACHER); picked[N,T] optional. */
int capb200_decode_sample(capb200_engine* e, const float* fc, const float* att, const float* mask, int B, int R, const capb200_sample_opts* opts,
                          const long long* tokens_in, long ld_tok, long long* seq, float* seq_logprobs, float* picked, void* stream);

/* Number of this library's kernel launches issued through the engine since creation (bench.py reports it). */
long capb200_engine_launch_count(const capb200_engine* e);

/* Optional device-side timing of the dense contractions (cudaEvent pairs recorded on the launching stream around every
 * GEMM launch).  ids: 0 fc_embed, 1 att_embed, 2 ctx2att, 3 fc->gate bias, 4 att_lstm gates, 5 h2att, 6 lang_lstm gates,
 * 7 logit, 8 newfc core.  read_profile synchronises the device and returns accumulated milliseconds, algorithmic FLOPs
 * (2*M*N*K) and launch counts per id; n must be >= 9. */
int capb200_engine_set_profiling(capb200_engine* e, int enable);
int capb200_engine_read_profile(capb200_engine* e, int reset, double* ms, double* flops, long* calls, int n);

/* ------------------------------------------------------------------------------------------------------------------
 * Transformer captioner (TransformerModel, captioning/models/TransformerModel.py:237-363)
 *   prologue = att_embed + N_enc encoder layers (TransformerModel.py:305-338); decode keeps a K/V cache per layer instead of
 *   re-running all t tokens each step (:351-363) -- identical results because the decoder mask is causal.
 * ---------------------------------------------------------------------------------------------------------------- */
#define CAPB200_TFM_MAX_LAYERS 8
typedef struct capb200_tfm_engine capb200_tfm_engine;
typedef struct {
    int vocab_size, d_model, d_ff, heads, n_enc, n_dec, att_feat_size, seq_length, numeric_mode;   /* seq_length 1..CAPB200_MAX_SEQ_LENGTH */
} capb200_tfm_cfg;
typedef struct { const float *q_w, *q_b, *k_w, *k_b, *v_w, *v_b, *o_w, *o_b; } capb200_mha_weights;          /* linears.0..3 */
typedef struct {
    capb200_mha_weights self_attn;
    const float *w1_w, *w1_b, *w2_w, *w2_b;                                                                   /* feed_forward.w_1 / w_2 */
    const float *ln0_a, *ln0_b, *ln1_a, *ln1_b;                                                               /* sublayer.{0,1}.norm.{a_2,b_2} */
} capb200_tfm_enc_layer;
typedef struct {
    capb200_mha_weights self_attn, src_attn;
    const float *w1_w, *w1_b, *w2_w, *w2_b;
    const float *ln0_a, *ln0_b, *ln1_a, *ln1_b, *ln2_a, *ln2_b;
} capb200_tfm_dec_layer;
typedef struct {
    const float *att_embed_w, *att_embed_b;                     /* att_embed.0 [D, F_att] */
    capb200_tfm_enc_layer enc[CAPB200_TFM_MAX_LAYERS];          /* model.encoder.layers.i */
    const float *enc_norm_a, *enc_norm_b;                       /* model.encoder.norm */
    capb200_tfm_dec_layer dec[CAPB200_TFM_MAX_LAYERS];          /* model.decoder.layers.i */
    const float *dec_norm_a, *dec_norm_b;                       /* model.decoder.norm */
    const float *lut, *pe;                                      /* model.tgt_embed.0.lut.weight [V+1, D]; model.tgt_embed.1.pe [1, 5000, D] */
    const float *gen_w, *gen_b;                                 /* model.generator.proj [V+1, D] */
} capb200_tfm_weights;

capb200_tfm_engine* capb200_tfm_create(const capb200_tfm_cfg* cfg);
void capb200_tfm_destroy(capb200_tfm_engine* e);
int capb200_tfm_bind_weights(capb200_tfm_engine* e, const capb200_tfm_weights* w, void* stream);
/* same contracts as capb200_decode_beam / capb200_beam_record_logprobs / capb200_decode_sample; fc features are unused */
int capb200_tfm_decode_beam(capb200_tfm_engine* e, const float* att, const float* mask, int B, int R, const capb200_beam_opts* opts, long long* seq,
                            float* seq_logprobs, long long* done_seq, int* done_len, float* done_p, float* done_raw, void* stream);
int capb200_tfm_beam_record_logprobs(capb200_tfm_engine* e, int image, int rank, float* dst, void* stream);
int capb200_tfm_decode_sample(capb200_tfm_engine* e, const float* att, const float* mask, int B, int R, const capb200_sample_opts* opts,
                              const long long* tokens_in, long ld_tok, long long* seq, float* seq_logprobs, float* picked, void* stream);
long capb200_tfm_launch_count(const capb200_tfm_engine* e);

/* ------------------------------------------------------------------------------------------------------------------
 * AoANet (AoAModel, captioning/models/AoAModel.py:188-226; configs/aoa.yml: refine=1, refine_aoa=1, use_ff=0,
 * decoder_type=AoA, use_multi_head=2, multi_head_scale=1, mean_feats=1)
 * ---------------------------------------------------------------------------------------------------------------- */
#define CAPB200_AOA_REFINER_LAYERS 6
typedef struct capb200_aoa_engine capb200_aoa_engine;
typedef struct {
    int vocab_size, input_encoding_size, rnn_size, heads, att_feat_size, seq_length, numeric_mode;   /* seq_length 1..CAPB200_MAX_SEQ_LENGTH */
} capb200_aoa_cfg;
typedef struct {
    const float *q_w, *q_b, *k_w, *k_b, *v_w, *v_b;   /* refiner.layers.i.self_attn.linears.{0,1,2} [H,H] */
    const float *aoa_w, *aoa_b;                       /* refiner.layers.i.self_attn.aoa_layer.0 [2H,2H] */
    const float *ln_a, *ln_b;                         /* refiner.layers.i.sublayer.0.norm.{a_2,b_2} */
} capb200_aoa_refiner_layer;
typedef struct {
    const float* embed;                               /* embed.0.weight [V+1,E] */
    const float *att_embed_w, *att_embed_b;           /* att_embed.0 [H,F_att] */
    capb200_aoa_refiner_layer refiner[CAPB200_AOA_REFINER_LAYERS];
    const float *refiner_norm_a, *refiner_norm_b;     /* refiner.norm */
    const float *ctx2att_w, *ctx2att_b;               /* ctx2att [2H,H] */
    const float *att_lstm_w_ih, *att_lstm_w_hh, *att_lstm_b_ih, *att_lstm_b_hh;   /* core.att_lstm [4H,E+H] [4H,H] */
    const float *attn_norm_a, *attn_norm_b;           /* core.attention.norm */
    const float *attn_q_w, *attn_q_b;                 /* core.attention.linears.0 [H,H] */
    const float *att2ctx_w, *att2ctx_b;               /* core.att2ctx.0 [2H,2H] */
    const float *logit_w, *logit_b;                   /* logit [V+1,H] */
} capb200_aoa_weights;

capb200_aoa_engine* capb200_aoa_create(const capb200_aoa_cfg* cfg);
void capb200_aoa_destroy(capb200_aoa_engine* e);
int capb200_aoa_bind_weights(capb200_aoa_engine* e, const capb200_aoa_weights* w, void* stream);
/* AoANet's logit head (AoAModel inherits AttModel's self.logit): as capb200_engine_set_logit_layers and the three after it */
int capb200_aoa_set_logit_layers(capb200_aoa_engine* e, int logit_layers);
int capb200_aoa_bind_logit_head(capb200_aoa_engine* e, const float* const* w, const float* const* b, void* stream);
int capb200_aoa_bind_logit_head_grads(capb200_aoa_engine* e, float* const* gw, float* const* gb);
int capb200_aoa_set_logit_dropout(capb200_aoa_engine* e, float p);
int capb200_aoa_decode_beam(capb200_aoa_engine* e, const float* att, const float* mask, int B, int R, const capb200_beam_opts* opts, long long* seq,
                            float* seq_logprobs, long long* done_seq, int* done_len, float* done_p, float* done_raw, void* stream);
int capb200_aoa_beam_record_logprobs(capb200_aoa_engine* e, int image, int rank, float* dst, void* stream);
/* same contract as capb200_decode_beam_diverse */
int capb200_aoa_decode_beam_diverse(capb200_aoa_engine* e, const float* att, const float* mask, int B, int R, const capb200_diverse_opts* opts,
                                    long long* seq, float* seq_logprobs, long long* done_seq, int* done_len, float* done_p, float* done_raw, void* stream);
int capb200_aoa_decode_sample(capb200_aoa_engine* e, const float* att, const float* mask, int B, int R, const capb200_sample_opts* opts,
                              const long long* tokens_in, long ld_tok, long long* seq, float* seq_logprobs, float* picked, void* stream);
long capb200_aoa_launch_count(const capb200_aoa_engine* e);

/* ------------------------------------------------------------------------------------------------------------------
 * Test-time ensemble (AttEnsemble, captioning/models/AttEnsemble.py): K members decode the same rows; every step mixes their word
 * distributions into log( sum_k softmax(z_k) * w_k / sum_k w_k ) (get_logprobs_state :50-58) and searches / samples on that row exactly as
 * a single model does on its log-probs.  Eval mode only; group_size 1.
 * ---------------------------------------------------------------------------------------------------------------- */
#define CAPB200_FAMILY_AOA 3              /* ensemble members only: `engine` is a capb200_aoa_engine */
#define CAPB200_ENSEMBLE_MAX_MEMBERS 8
typedef struct {
    int family;       /* CAPB200_FAMILY_UPDOWN / NEWFC / ATT2IN2 (engine: capb200_engine*) or CAPB200_FAMILY_AOA (engine: capb200_aoa_engine*) */
    void* engine;     /* bound; every member on the current device, with the first member's vocab_size and seq_length */
    float weight;     /* >= 0, not all zero */
} capb200_ensemble_member;
/* Owns the ensemble's decode state: the [K, rows, V+1] member logits, beam records and the CUDA graph of the beam loop.  Member engines
 * stay owned by the caller and may also decode on their own between ensemble calls. */
typedef struct capb200_ensemble capb200_ensemble;
capb200_ensemble* capb200_ensemble_create(void);
void capb200_ensemble_destroy(capb200_ensemble* s);
/* Same contract as capb200_decode_beam, over K = 1..CAPB200_ENSEMBLE_MAX_MEMBERS members.  fc may be NULL when no member reads it (AoA,
 * Att2in2), att when none attends (NewFC only).  Members, K and weights are checked before any device work. */
int capb200_ensemble_decode_beam(capb200_ensemble* s, const capb200_ensemble_member* members, int K, const float* fc, const float* att,
                                 const float* mask, int B, int R, const capb200_beam_opts* opts, long long* seq, float* seq_logprobs,
                                 long long* done_seq, int* done_len, float* done_p, float* done_raw, void* stream);
/* done_beams[image][rank]['logps'] of the last capb200_ensemble_decode_beam call (contract of capb200_beam_record_logprobs) */
int capb200_ensemble_beam_record_logprobs(capb200_ensemble* s, int image, int rank, float* dst, void* stream);
/* Same contract as capb200_decode_sample: greedy, multinomial / top-k / nucleus sampling, forced replay and teacher forcing. */
int capb200_ensemble_decode_sample(capb200_ensemble* s, const capb200_ensemble_member* members, int K, const float* fc, const float* att,
                                   const float* mask, int B, int R, const capb200_sample_opts* opts, const long long* tokens_in, long ld_tok,
                                   long long* seq, float* seq_logprobs, float* picked, void* stream);
/* Kernel launches of the ensemble's decodes (its own and its members' on its behalf, replayed graph launches included). */
long capb200_ensemble_launch_count(const capb200_ensemble* s);

/* ------------------------------------------------------------------------------------------------------------------
 * SCST reward and criterion
 * ---------------------------------------------------------------------------------------------------------------- */
/* Document-frequency table in the scripts/prepro_ngrams.py format, flattened: keys[n,4] int32 token ids padded with -1,
 * df[n] float64, ref_len = number of reference images (ciderD_scorer.py:108-111).  Host pointers; synchronous. */
capb200_cider_table* capb200_cider_table_create(const int* keys, const double* df, long n, double ref_len, void* stream);
void capb200_cider_table_destroy(capb200_cider_table* t);
/* Corpus document frequencies (init_scorer('corpus') -> CiderD(df='corpus'), ciderD_scorer.py:143-147,182-186,210-216): no pickle; every
 * reward call that reads the table (the entry points below and every family's SCST / new_self_critical step) first rebuilds it on the device
 * from its own references, in three kernels inside the same stream (and step graph).  df[ngram] counts the scored hypotheses (crefs entries)
 * whose reference set holds the n-gram -- each image's distinct n-grams count once per hypothesis of the image: n + 1 with greedy captions,
 * n without -- and ref_len = log(number of hypotheses).  Before a call, reserve room for its references: n_refs rows of L tokens (growing
 * synchronises the device and moves the slots, which a captured step graph notices).  A call with more reference rows than reserved
 * undercounts instead of overflowing the table. */
capb200_cider_table* capb200_cider_corpus_table_create(void);
int capb200_cider_table_reserve(capb200_cider_table* t, long n_refs, int L);
int capb200_cider_table_is_corpus(const capb200_cider_table* t);

/* get_self_critical_reward (captioning/utils/rewards.py:41-81) with CIDEr-D only:
 * sampled[S,T], greedy[B,T] int64 device; refs[n_refs_total,L] int32 device (0 padded), ref_offsets[B+1] int32 device;
 * T and L up to CAPB200_MAX_SEQ_LENGTH (every reward entry point below takes the same bound; a caption ends at its first 0);
 * scores[S+B] float64 device (CIDEr-D of every hypothesis); reward[S,T] fp32 = score(sample) - score(greedy of its image). */
int capb200_self_critical_reward(const capb200_cider_table* t, const long long* sampled, int S, const long long* greedy, int B, int T,
                                 const int* refs, const int* ref_offsets, int L, double* scores, float* reward, void* stream);

/* get_scores (captioning/utils/rewards.py:83-114) with cider_reward_weight = 1: CIDEr-D of S = B*n sampled captions against their
 * image's references -> scores[S] float64.  reward (optional, [S,T] fp32): score minus the mean score of the image's other samples,
 * the per-token weight of the 'new_self_critical' structure loss (losses.py:168-187). */
int capb200_cider_scores(const capb200_cider_table* t, const long long* sampled, int S, int B, int T, const int* refs, const int* ref_offsets,
                         int L, double* scores, float* reward, void* stream);

/* Weights of the two reward terms (opts.py:169-172): score = cider * CIDEr-D + bleu * BLEU-4 (rewards.py:63-74, :100-112).  A term is
 * computed only when its weight is > 0; otherwise it contributes weight * 0.  A NULL pointer to this struct means {1, 0}, the CIDEr-D reward. */
typedef struct {
    double cider;
    double bleu;
} capb200_reward_weights;

/* BLEU-4 of every hypothesis against its image's references: the per-sentence bleu_list[3] of Bleu(4).compute_score (closest reference
 * length, coco-caption/pycocoevalcap/bleu/bleu_scorer.py), float64.  Hypotheses sampled[S,T] (image i / (S/B)) and, if greedy[B,T] is not
 * NULL, greedy rows S..S+B-1; refs / ref_offsets / L as in capb200_self_critical_reward.  scores[S (+B)].  An image without references
 * scores 0 (the reference asserts that every image has one). */
int capb200_bleu4_scores(const long long* sampled, int S, const long long* greedy, int B, int T, const int* refs, const int* ref_offsets, int L,
                         double* scores, void* stream);

/* get_self_critical_reward (greedy != NULL) and get_scores (greedy == NULL) with both reward terms.  scores[S (+B)] float64: the weighted
 * score of every hypothesis.  bleu_scores[S (+B)] float64: BLEU-4 of every hypothesis (required when w->bleu > 0, else ignored).  t may be
 * NULL when w->cider <= 0.  reward (optional, [S,T] fp32): score(sample) - score(greedy of its image) in float64 then cast, or -- without
 * greedy -- the leave-one-out reward of capb200_cider_scores over the fp32-cast scores.  With w = NULL or {1, 0} the result equals
 * capb200_self_critical_reward / capb200_cider_scores. */
int capb200_weighted_reward(const capb200_cider_table* t, const capb200_reward_weights* w, const long long* sampled, int S, const long long* greedy,
                            int B, int T, const int* refs, const int* ref_offsets, int L, double* scores, double* bleu_scores, float* reward,
                            void* stream);

/* RewardCriterion.forward (captioning/modules/losses.py:22-37). logprobs[N,T,V1]; seq[N,T] int64; reward[N,T].
 * loss_mean[1], loss_rows[N] (reduction 'none'), mask_sum[1]; any output may be NULL. */
int capb200_reward_criterion_forward(const float* logprobs, const long long* seq, const float* reward, int N, int T, int V1, float* loss_mean,
                                     float* loss_rows, float* mask_sum, void* stream);
/* d loss_mean / d logprobs, scaled by `upstream`; grad[N,T,V1] must be zero-filled by the caller. */
int capb200_reward_criterion_backward(const long long* seq, const float* reward, int N, int T, int V1, const float* mask_sum, float upstream,
                                      float* grad, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Diversity of caption sets (captioning/utils/rewards.py:116-138 get_self_cider_scores, captioning/utils/eval_multi.py:121-217)
 * seqs[n_images * n, T] int64 device: n consecutive captions per image, 2 <= n <= 32, T <= 64.  Nothing is allocated; every output is
 * float64 device memory unless stated.
 * ---------------------------------------------------------------------------------------------------------------- */
/* Self-CIDEr: out_mat[n_images, n, n] = CiderScorer.my_get_self_cider (plain CIDEr: tf-idf cosine per order, mean over orders 1..4, x 10)
 * with the document frequencies and ref_len of `t`; an n-gram the table does not hold has df 0.  with_eos = 1 keeps each caption through
 * its first 0 (array_to_str, the reward form), 0 stops before it (the decoded words of eval_self_cider).  out_score[n_images] = the
 * eigenvalue diversity of out_mat, as capb200_self_cider_div computes it.  A corpus table is refused. */
int capb200_self_cider(const capb200_cider_table* t, const long long* seqs, int n_images, int n, int T, int with_eos, double* out_mat,
                       double* out_score, void* stream);
/* out_score[i] = -log(sqrt(l_max) / sum_k sqrt(l_k)) / log(n) over the eigenvalues l of mat[i] / 10 clipped at 0 (rewards.py:130-133);
 * like numpy's eigvalsh, only the lower triangle of mat[n_images, n, n] is read.  All-zero eigenvalues give nan, as in the reference. */
int capb200_self_cider_div(const double* mat, int n_images, int n, double* out_score, void* stream);
/* Div-n and mutual BLEU over the words of each caption (the ids before its first 0), ids in [1, V1):
 *   out_div1[n_images], out_div2[n_images]   distinct uni- / bigrams of the image's captions / (1e-6 + words) (div_utils.compute_div_n)
 *   out_gdiv1[1]                             distinct words over every caption (compute_global_div_n), -1 if an id is outside [1, V1)
 *   out_mbleu[n, 4]                          corpus BLEU-1..4 of leave-one-out round j: caption j of every image against its other n - 1
 *   out_bleu2[n_images, n]                   per-sentence BLEU-2 of caption j against the image's other captions (Bleu(4) scores[1])
 *   out_bleu_stats[n_images, n, 6] int32     correct 1..4-grams, length and closest reference length of each caption in its round */
int capb200_div_stats(const long long* seqs, int n_images, int n, int T, int V1, double* out_div1, double* out_div2, double* out_gdiv1,
                      double* out_mbleu, double* out_bleu2, int* out_bleu_stats, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Language evaluation: coco-caption's Bleu(4), Rouge() and Cider() (coco-caption/pycocoevalcap) over token ids
 * seqs[n_images * per_image, T] int64 device: per_image consecutive captions per image; a caption is its ids before the first 0, scored
 * as the string of those ids joined by single spaces.  refs / ref_offsets / L as in capb200_self_critical_reward, each reference cut before
 * its first 0.  T and L between 1 and CAPB200_MAX_SEQ_LENGTH.  These are not the official COCO numbers: there is no PTB tokenization of the
 * annotation text, and the references are the dataset's label rows (truncated at max_length, rare words UNK).
 * ---------------------------------------------------------------------------------------------------------------- */
/* Outputs, float64 device memory:
 *   out_bleu[S, 4]                  each caption's per-sentence BLEU-1..4 (Bleu(4) bleu_list, closest reference length)
 *   out_corpus_bleu[per_image, 4]   corpus BLEU-1..4 of round j: caption j of every image (Bleu(4)'s overall score of that round)
 *   out_rouge[S]                    ROUGE-L (beta = 1.2; an empty caption is one empty word, as str.split(" ") makes it)
 *   out_cider[S]                    CIDEr: document frequencies count each image once, ref_len = log(n_images), whatever per_image is
 * ws_stats[S, 6] int32 device: scratch (correct 1..4-grams, length and closest reference length of each caption).  `t` is a corpus table
 * (capb200_cider_corpus_table_create), reserved here for the references; only its first call at a given size allocates.  The B + 1 offsets
 * are read back (the stream is synchronised) and an image without references is refused before any launch. */
int capb200_coco_scores(capb200_cider_table* t, const long long* seqs, int n_images, int per_image, int T, const int* refs, const int* ref_offsets,
                        int L, double* out_bleu, double* out_corpus_bleu, double* out_rouge, double* out_cider, int* ws_stats, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * One self-critical training step of the UpDown model (LossWrapper.forward with sc_flag, loss_wrapper.py:56-73, plus the
 * loss.backward() of tools/train.py:189): eval-mode greedy baseline, train-mode multinomial samples (dropout on, AttModel.py:74-88,
 * :637), self-critical reward (CIDEr-D, or weighted CIDEr-D + BLEU-4 with opts->reward_weights), RewardCriterion, then back-propagation
 * through time into every parameter gradient.
 * ---------------------------------------------------------------------------------------------------------------- */
/* How a fused self-critical step draws its words: LossWrapper's train_sample_method (the train-mode samples, loss_wrapper.py:63-67) and
 * sc_sample_method (the eval-mode baseline, :57-62), both at temperature 1 for the baseline and opts->temperature for the samples.  Methods
 * are CAPB200_SAMPLE_GREEDY, _MULTINOMIAL, _TOPK (top = k >= 1) and _TOPP (0 < top < 1), drawn as capb200_decode_sample draws them; 'gumbel'
 * is a multinomial draw at temperature 1.  The criterion and the gradient always use the full log-softmax row (AttModel.py:337,347).  The
 * baseline draws from its own Philox key, derived from opts->seed, so a replayed step graph draws fresh baseline captions too.  A NULL
 * pointer to this struct means {MULTINOMIAL, 0, GREEDY, 0, NULL}.  A sampled baseline needs CAPB200_BASELINE_GREEDY. */
typedef struct {
    int train_method;
    float train_top;
    int baseline_method;
    float baseline_top;
    const long long* forced_baseline;   /* optional [B, T] int64 device: replay these baseline captions instead of drawing them (parity checks) */
} capb200_sampler_opts;
typedef struct {
    int sample_n;              /* opt.train_sample_n */
    float temperature;
    unsigned long long seed;   /* Philox key of the sampler and of the dropout masks */
    float drop_prob;           /* drop_prob_lm; 0 disables dropout */
    float upstream;            /* d(total loss)/d(this loss), normally 1 */
    int baseline;              /* CAPB200_BASELINE_GREEDY (self-critical, loss_wrapper.py:56-73) or CAPB200_BASELINE_LEAVE_ONE_OUT
                                  (structure loss 'new_self_critical', losses.py:168-187: no greedy decode, greedy_seq may be NULL) */
    const long long* forced_tokens; /* optional [B*sample_n, T] int64 device: replay these samples instead of drawing them (parity
                                  checks against the reference's own multinomial draw); NULL = sample */
    const float* att_masks;    /* optional [B, R] fp32 device (1 = valid region): variable region counts (AttModel.py:44-49,106-112,742-744;
                                  dataloader.py:230-241); the caller has clipped R to the longest valid length; NULL = all regions valid */
    int keep_rows;             /* drop_worst (tools/train.py:187-191): 0 = reduction 'mean'; k > 0 = the criterion runs with reduction 'none' (one loss per
                                  caption row) and the k rows with the smallest loss are averaged: loss[0] = that mean, gradients accordingly */
    float* row_loss;           /* optional [rows] output of the per-row losses (what LossWrapper returns as out['loss'] under drop_worst_flag) */
    const capb200_sampler_opts* sampler; /* optional, read during the call: the train and baseline samplers; NULL = multinomial samples and the
                                  greedy baseline.  The autograd entry points (*_scst_vjp) refuse it */
    const capb200_reward_weights* reward_weights; /* optional, read during the call: the reward is cider * CIDEr-D + bleu * BLEU-4 as
                                  capb200_weighted_reward computes it; NULL = CIDEr-D only (weight 1) */
} capb200_scst_opts;
#define CAPB200_BASELINE_GREEDY 0
#define CAPB200_BASELINE_LEAVE_ONE_OUT 1
/* Gradient buffers, one per capb200_weights field (same shapes, fp32, device); every one is OVERWRITTEN. */
typedef struct {
    float* embed;
    float *fc_embed_w, *fc_embed_b, *att_embed_w, *att_embed_b, *ctx2att_w, *ctx2att_b, *logit_w, *logit_b;
    float *att_lstm_w_ih, *att_lstm_w_hh, *att_lstm_b_ih, *att_lstm_b_hh, *lang_lstm_w_ih, *lang_lstm_w_hh, *lang_lstm_b_ih, *lang_lstm_b_hh;
    float *h2att_w, *h2att_b, *alpha_w, *alpha_b;
} capb200_updown_grads;
/* fc[B,F_fc], att[B,R,F_att] (opts->att_masks for variable region counts); refs as in capb200_self_critical_reward.
 * Outputs: sample_seq[B*n,T] int64, greedy_seq[B,T] int64, sample_logprobs[B*n,T,V+1] (caller zero-fills), reward[B*n,T], loss[1].
 * Execution: the whole step (~900-4900 launches, none of them data dependent) is captured into ONE CUDA graph the second time a configuration
 * -- shapes, every pointer argument, every option except the seed -- is seen, and replayed afterwards (the *_scst_step entry points of every
 * family; CAPB200_SCST_GRAPH=0 disables it).  For that the step runs on an engine-owned stream that first waits for `stream` and that
 * `stream` is made to wait for before the call returns; the features (and the region mask) are copied into an engine-owned staging buffer, so
 * they may live anywhere, while refs / ref_offsets / the output and gradient buffers should keep their addresses from step to step (a changed
 * address is a new configuration: one eager step, one capture).  A replay draws new samples and masks from opts->seed exactly as the eager
 * step would (the seed reaches the kernels through a device-side salt), so results do not depend on whether a step was replayed. */
int capb200_updown_scst_step(capb200_engine* e, const float* fc, const float* att, int B, int R, const capb200_scst_opts* opts,
                             const capb200_cider_table* table, const int* refs, const int* ref_offsets, int L, const capb200_updown_grads* grads,
                             long long* sample_seq, long long* greedy_seq, float* sample_logprobs, float* reward, float* loss, void* stream);
/* ------------------------------------------------------------------------------------------------------------------
 * One cross-entropy (XE) training step of the UpDown model: the teacher-forced AttModel._forward (AttModel.py:126-164; train mode,
 * dropout on, no scheduled sampling) over labels[..., :-1], LanguageModelCriterion or LabelSmoothing (losses.py:204-265) against
 * labels[..., 1:] / masks[..., 1:] with reduction 'mean' (loss_wrapper.py:54-55), and back-propagation through time.
 * ---------------------------------------------------------------------------------------------------------------- */
typedef struct {
    int seq_per_img;           /* label rows per image (the reference repeats the features, utils.repeat_tensors) */
    int steps;                 /* columns actually evaluated: the reference stops at the first column i >= 1 whose tokens are all 0 */
    unsigned long long seed;   /* Philox key of the dropout masks */
    float drop_prob;
    float label_smoothing;     /* 0 = LanguageModelCriterion, > 0 = LabelSmoothing(smoothing) */
    float upstream;
    const float* att_masks;    /* optional [B, R] region mask, see capb200_scst_opts */
    float ss_prob;             /* scheduled sampling (AttModel.py:145-154): from the second step on, each row's input word is drawn from the model's
                                  previous prediction with this probability; 0 = teacher forcing */
    long long* tokens_used;    /* optional [N, label_cols-1] int64: the words actually fed (labels, or the draws where scheduled sampling hit) */
    int keep_rows;             /* drop_worst (tools/train.py:187-191): 0 = reduction 'mean'; k > 0 = the criterion runs with reduction 'none' (one loss per
                                  caption row) and the k rows with the smallest loss are averaged: loss[0] = that mean, gradients accordingly */
    float* row_loss;           /* optional [rows] output of the per-row losses (what LossWrapper returns as out['loss'] under drop_worst_flag) */
} capb200_xe_opts;
/* labels[N, label_cols] int64 (column 0 = BOS = 0), masks[N, label_cols] fp32, N = B * seq_per_img.
 * Outputs: logprobs[N, label_cols-1, V+1] (caller zero-fills; columns >= steps stay zero), loss[1], every grads buffer overwritten. */
int capb200_updown_xe_step(capb200_engine* e, const float* fc, const float* att, int B, int R, const capb200_xe_opts* opts, const long long* labels,
                           const float* masks, int label_cols, const capb200_updown_grads* grads, float* logprobs, float* loss, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Training steps of the Att2in2 model (Att2in2Core, AttModel.py:770-790), same contracts as the UpDown steps above: an engine of
 * CAPB200_FAMILY_ATT2IN2, the fc features are ignored (may be NULL), the options mean what they mean for UpDown (greedy or leave-one-out
 * baseline, forced tokens, region masks, keep_rows / row_loss, scheduled sampling with tokens_used, label smoothing), dropout sites
 * 1 att_embed, 2 word embedding, 3 core output (replayable through capb200_dropout_mask), the whole SCST step captured into one CUDA graph as
 * capb200_updown_scst_step describes.  Gradient groups: see capb200_engine_set_grad_events.
 * ---------------------------------------------------------------------------------------------------------------- */
/* Gradient buffers of the 17 Att2in2 parameters (same shapes as the capb200_weights fields, fp32, device); every one is OVERWRITTEN. */
typedef struct {
    float* embed;
    float *att_embed_w, *att_embed_b, *ctx2att_w, *ctx2att_b, *logit_w, *logit_b;
    float *h2att_w, *h2att_b, *alpha_w, *alpha_b;
    float *i2h_w, *i2h_b, *h2h_w, *h2h_b, *a2c_w, *a2c_b;
} capb200_att2in2_grads;
int capb200_att2in2_scst_step(capb200_engine* e, const float* fc, const float* att, int B, int R, const capb200_scst_opts* opts,
                              const capb200_cider_table* table, const int* refs, const int* ref_offsets, int L, const capb200_att2in2_grads* grads,
                              long long* sample_seq, long long* greedy_seq, float* sample_logprobs, float* reward, float* loss, void* stream);
int capb200_att2in2_xe_step(capb200_engine* e, const float* fc, const float* att, int B, int R, const capb200_xe_opts* opts, const long long* labels,
                            const float* masks, int label_cols, const capb200_att2in2_grads* grads, float* logprobs, float* loss, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Training steps of the NewFC model (NewFCModel, AttModel.py:904-945, with FCModel.LSTMCore, FCModel.py:13-42), same contracts as the UpDown
 * steps above: an engine of CAPB200_FAMILY_NEWFC; the options mean what they mean for UpDown (greedy or leave-one-out baseline, forced tokens,
 * keep_rows / row_loss, scheduled sampling with tokens_used, label smoothing).  The model reads the fc features only: `att` is ignored (NULL
 * with R = 0 is fine) and a non-NULL opts->att_masks is refused.  The core first consumes fc_embed(fc) from a zero state (once per image),
 * then <bos> and the words; the only dropout is site 3, the core output (replayable through capb200_dropout_mask).  The SCST step is captured
 * into one CUDA graph as capb200_updown_scst_step describes.  Gradient groups: see capb200_engine_set_grad_events.
 * ---------------------------------------------------------------------------------------------------------------- */
/* Gradient buffers of the 9 NewFC parameters (same shapes as the capb200_weights fields, fp32, device); every one is OVERWRITTEN. */
typedef struct {
    float* embed;
    float *fc_embed_w, *fc_embed_b, *logit_w, *logit_b;
    float *i2h_w, *i2h_b, *h2h_w, *h2h_b;
} capb200_newfc_grads;
int capb200_newfc_scst_step(capb200_engine* e, const float* fc, const float* att, int B, int R, const capb200_scst_opts* opts,
                            const capb200_cider_table* table, const int* refs, const int* ref_offsets, int L, const capb200_newfc_grads* grads,
                            long long* sample_seq, long long* greedy_seq, float* sample_logprobs, float* reward, float* loss, void* stream);
int capb200_newfc_xe_step(capb200_engine* e, const float* fc, const float* att, int B, int R, const capb200_xe_opts* opts, const long long* labels,
                          const float* masks, int label_cols, const capb200_newfc_grads* grads, float* logprobs, float* loss, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * One self-critical training step of the AoANet model (BASELINE configs[3]): LossWrapper.forward with sc_flag (loss_wrapper.py:56-73)
 * over AoAModel (refiner + AoA decoder, AoAModel.py:56-226) in train mode, and its backward.  Dropout sites (replayable through
 * capb200_dropout_mask with the same seed): 1 att_embed [B*R,H]; 2 word embedding at `step` [N,E]; 3 core output at `step` [N,H];
 * 4 ctx_drop at `step` [N,H]; 5 decoder attention probabilities at `step` [N,heads,R]; 10+l refiner attention probabilities
 * [B,heads,R,R]; 20+l AoA-layer input [B*R,2H]; 30+l refiner SublayerConnection [B*R,H]   (l = refiner layer 0..5).
 * ---------------------------------------------------------------------------------------------------------------- */
typedef struct {
    int sample_n;
    float temperature;
    unsigned long long seed;
    float upstream;
    int baseline;              /* CAPB200_BASELINE_* */
    float drop_prob_lm;        /* att_embed, word embedding, ctx_drop, out_drop (opt.drop_prob_lm) */
    float drop_attn;           /* MultiHeadedDotAttention dropout on the probabilities (0.1, AoAModel.py:18) */
    float drop_aoa;            /* dropout_aoa (0.3) */
    float drop_sublayer;       /* refiner SublayerConnection (0.1, AoAModel.py:119) */
    int ctx_drop;              /* opt.ctx_drop */
    const long long* forced_tokens; /* optional [B*sample_n, T] int64 device: replay these samples (see capb200_scst_opts) */
    const float* att_masks;    /* optional [B, R] region mask (refiner self-attention keys, masked mean pooling AoAModel.py:216-219, decoder
                                  attention keys) */
    int keep_rows;             /* drop_worst (tools/train.py:187-191): 0 = reduction 'mean'; k > 0 = the criterion runs with reduction 'none' (one loss per
                                  caption row) and the k rows with the smallest loss are averaged: loss[0] = that mean, gradients accordingly */
    float* row_loss;           /* optional [rows] output of the per-row losses (what LossWrapper returns as out['loss'] under drop_worst_flag) */
    const capb200_sampler_opts* sampler;          /* optional samplers, see capb200_scst_opts; NULL = multinomial + greedy baseline */
    const capb200_reward_weights* reward_weights; /* optional reward weights, see capb200_scst_opts; NULL = CIDEr-D only */
} capb200_aoa_scst_opts;
/* Gradient buffers, laid out field by field like the weights struct above: parameter shapes, fp32, device; every one is OVERWRITTEN. */
typedef struct {
    float *q_w, *q_b, *k_w, *k_b, *v_w, *v_b, *aoa_w, *aoa_b, *ln_a, *ln_b;
} capb200_aoa_refiner_layer_grads;
typedef struct {
    float* embed;
    float *att_embed_w, *att_embed_b;
    capb200_aoa_refiner_layer_grads refiner[CAPB200_AOA_REFINER_LAYERS];
    float *refiner_norm_a, *refiner_norm_b;
    float *ctx2att_w, *ctx2att_b;
    float *att_lstm_w_ih, *att_lstm_w_hh, *att_lstm_b_ih, *att_lstm_b_hh;
    float *attn_norm_a, *attn_norm_b;
    float *attn_q_w, *attn_q_b;
    float *att2ctx_w, *att2ctx_b;
    float *logit_w, *logit_b;
} capb200_aoa_grads;
/* att[B,R,F_att] (opts->att_masks for variable region counts); outputs as in capb200_updown_scst_step. */
int capb200_aoa_scst_step(capb200_aoa_engine* e, const float* att, int B, int R, const capb200_aoa_scst_opts* opts, const capb200_cider_table* table,
                          const int* refs, const int* ref_offsets, int L, const capb200_aoa_grads* grads, long long* sample_seq, long long* greedy_seq,
                          float* sample_logprobs, float* reward, float* loss, void* stream);

/* One cross-entropy training step of AoANet (teacher-forced AttModel._forward over AoAModel in train mode + LanguageModelCriterion /
 * LabelSmoothing + backward); arguments as capb200_updown_xe_step, dropout sites as capb200_aoa_scst_step. */
typedef struct {
    int seq_per_img;
    int steps;                 /* columns actually evaluated (early break of AttModel.py:158-159) */
    unsigned long long seed;
    float label_smoothing;
    float upstream;
    float drop_prob_lm, drop_attn, drop_aoa, drop_sublayer;
    int ctx_drop;
    const float* att_masks;    /* optional [B, R] region mask */
    float ss_prob;             /* scheduled sampling, see capb200_xe_opts */
    long long* tokens_used;
    int keep_rows;             /* drop_worst (tools/train.py:187-191): 0 = reduction 'mean'; k > 0 = the criterion runs with reduction 'none' (one loss per
                                  caption row) and the k rows with the smallest loss are averaged: loss[0] = that mean, gradients accordingly */
    float* row_loss;           /* optional [rows] output of the per-row losses (what LossWrapper returns as out['loss'] under drop_worst_flag) */
} capb200_aoa_xe_opts;
int capb200_aoa_xe_step(capb200_aoa_engine* e, const float* att, int B, int R, const capb200_aoa_xe_opts* opts, const long long* labels,
                        const float* masks, int label_cols, const capb200_aoa_grads* grads, float* logprobs, float* loss, void* stream);

/* Gradient-group events for an overlapped data-parallel all-reduce (tools/train_pl.py:479: DDP buckets the reference's gradients the
 * same way).  A training step finishes its gradient buffers in a fixed order of groups; after the last write of group k it records
 * events[k] (cudaEvent_t, caller-owned) on the step's stream, so a communication stream can all-reduce group k while the rest of the
 * backward pass still runs.  n = 0 or events = NULL switches the recording off.  Groups:
 *   UpDown, Att2in2 and NewFC (capb200_engine_set_grad_events, n <= 2): 0 logit.{weight,bias}; 1 every other parameter.
 *   AoANet (capb200_aoa_set_grad_events, n <= 10):  0 logit; 1 decoder (att2ctx, attention q-projection and norm, att_lstm) + embed;
 *           2 ctx2att + refiner.norm; 3..8 refiner layers 5..0; 9 att_embed. */
int capb200_engine_set_grad_events(capb200_engine* e, void* const* events, int n);
int capb200_aoa_set_grad_events(capb200_aoa_engine* e, void* const* events, int n);

/* The dropout keep/scale mask (0 or 1/(1-p)) of one site and step, for tests that replay it in the oracle:
 * site 0 = fc_embed [B,H], 1 = att_embed [B*R,H], 2 = word embedding at `step` [N,E], 3 = core output at `step` [N,H].
 * (Att2in2 has no site 0: it has no fc_embed.  NewFC has site 3 only: its embeddings are a bare nn.Embedding / nn.Linear.) */
int capb200_dropout_mask(float* mask, long n, unsigned long long seed, int site, int step, float p, void* stream);

/* Multi-head attention operations of the AoANet refiner / Transformer encoder and of the decoders' attention over the regions, for tests.
 * `form`: 0 picks the kernel as the training steps and the decoder do (the staged kernel when its shared-memory footprint fits in 200 KB,
 * else the key-tiled one), 1 forces the staged kernel (an error where it does not fit), 2 forces the key-tiled kernel (head width a multiple
 * of 4, at most 256).  Head h of a row is columns [h*dk, (h+1)*dk); scale 1/sqrt(dk); mask [B, ld_mask] (0 = masked key) or NULL.
 * Dropout on the probabilities uses element ((b*heads + h)*R + i)*R + r at step 0 of `site` (self-attention) and item*R + r with
 * item = (row within its time block)*heads + h at step `step` + time block (cross-attention): capb200_dropout_mask replays both.
 *   capb200_mha_forward        out = softmax(q k^T / sqrt(dk)) v over the R regions of each of B images, rows image-major [B*R, ld];
 *                              train = 0: the decode form (no dropout; seed, site and p unused), 1: the training form with dropout p
 *   capb200_mha_self_backward  dq, dkey, dval (written, pitch ld_d; dq must not alias an input) of capb200_mha_forward(train = 1)
 *   capb200_mha_cross_backward rows TIME-major: row = t*(B*rpi) + b*rpi + j for t < n_steps; keys / values [B*R, ld_kv]; probs [rows*heads, R]
 *                              the saved probabilities before dropout; dq written, dk / dv ADDED into [B*R, ld_dkv]
 * Return 0 or 1 (capb200_last_error). */
int capb200_mha_forward(int form, int train, int B, int R, int heads, int dk, const float* q, const float* k, const float* v, long ld, const float* mask,
                        long ld_mask, unsigned long long seed, int site, float p, float* out, long ld_out, void* stream);
int capb200_mha_self_backward(int form, int B, int R, int heads, int dk, const float* q, const float* k, const float* v, long ld, const float* mask,
                              long ld_mask, unsigned long long seed, int site, float p, const float* d_out, long ld_do, float* dq, float* dkey, float* dval,
                              long ld_d, void* stream);
int capb200_mha_cross_backward(int form, int B, int rpi, int n_steps, int heads, int dk, int R, const float* q, long ld_q, const float* kk, const float* vv,
                               long ld_kv, unsigned long long seed, int site, int step, float p, const float* probs, const float* d_out, long ld_do, float* dq,
                               long ld_dq, float* dkk, float* dvv, long ld_dkv, void* stream);

/* The Transformer decoder's causal self-attention in training, for tests: B sequences of T positions, rows image-major [B*T, ld]; key r is
 * visible to query i iff r <= i and key_mask[b, r] != 0 (key_mask [B, ld_mask] or NULL).  Dropout element ((b*heads + h)*T + i)*T + r at
 * step 0 of `site`.  `form` as for capb200_mha_forward; the key-tiled form skips the key tiles past each query tile.
 *   capb200_mha_causal_forward   out rows of the queries [q_lo, q_hi) (every key up to the query is read)
 *   capb200_mha_causal_backward  dq, dkey, dval of capb200_mha_causal_forward over all T queries (dq must not alias an input) */
int capb200_mha_causal_forward(int form, int B, int T, int q_lo, int q_hi, int heads, int dk, const float* q, const float* k, const float* v, long ld,
                               const float* key_mask, long ld_mask, unsigned long long seed, int site, float p, float* out, long ld_out, void* stream);
int capb200_mha_causal_backward(int form, int B, int T, int heads, int dk, const float* q, const float* k, const float* v, long ld, const float* key_mask,
                                long ld_mask, unsigned long long seed, int site, float p, const float* d_out, long ld_do, float* dq, float* dkey, float* dval,
                                long ld_d, void* stream);

/* The Transformer's decoder self-attention at step t, for tests.  qkv [rows, ld_qkv] holds this step's q | k | v (D = heads*dk columns
 * each); kcache / vcache [t+1][step_stride] hold the keys / values of positions < t at row * ld_c (+ head*dk) and receive this step's k, v;
 * anc [rows, ld_anc] the row whose cache entry position s < t reads (beam search), or NULL for the row itself; labels [rows, ld_lab] int64
 * or NULL: teacher forcing masks positions s > 0 whose label is 0.  out [rows, ld_out].  form 0 picks the kernel as the decoder does (one
 * lane per position for t < 32, the chunked online softmax beyond), 1 forces the first (t < 32 only), 2 the second (head width <= 256). */
int capb200_tfm_dec_self_attention(int form, int rows, int heads, int dk, int t, const float* qkv, long ld_qkv, float* kcache, float* vcache,
                                   long step_stride, long ld_c, const int* anc, long ld_anc, const long long* labels, long ld_lab, float* out, long ld_out,
                                   void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Training steps of the Transformer captioner (TransformerModel.py:262-363 under LossWrapper, loss_wrapper.py:25-73, + loss.backward()).
 *   capb200_tfm_xe_step    the teacher-forced TransformerModel._forward (:340-348: one pass over all label_cols - 1 positions; keys that
 *                          are pad / eos are masked, position 0 never, :323-328) + LanguageModelCriterion / LabelSmoothing + backward;
 *                          labels / masks / logprobs / loss as capb200_updown_xe_step (logprobs [N, label_cols - 1, V+1], all positions)
 *   capb200_tfm_scst_step  eval-mode greedy baseline (or leave-one-out), train-mode multinomial samples, CIDEr-D reward, RewardCriterion,
 *                          backward; arguments as capb200_aoa_scst_step
 * The gradient table has the field layout of the weight table (every pointer is written; `pe` is a buffer and is ignored).
 * dropout = the Transformer's own rate (attention probabilities, SublayerConnections, feed-forward, positional encoding: 0.1);
 * drop_prob_lm = att_embed's Dropout.  Replayable through capb200_dropout_mask(seed, site, step, ...) with, per site, step = the position t
 * and the element index n * cols + c for decoder tensors [N, cols] (encoder tensors [B*R, cols]: step 0): 1 att_embed; 2 target embedding;
 * encoder layer l: 10+l attention probabilities [B, heads, R, R], 20+l / 40+l SublayerConnections, 30+l feed-forward hidden;
 * decoder layer l: 50+l self-attention probabilities (step 0, index ((n*heads + h)*(T+2) + t)*(T+2) + s), 60+l / 80+l / 100+l
 * SublayerConnections, 70+l source-attention probabilities [N, heads, R] at step t, 90+l feed-forward hidden.
 * The encoder runs once per image (the reference's _forward runs it once per caption: same values, seq_per_img x the work).
 * ---------------------------------------------------------------------------------------------------------------- */
typedef struct { float *q_w, *q_b, *k_w, *k_b, *v_w, *v_b, *o_w, *o_b; } capb200_mha_grads;
typedef struct {
    capb200_mha_grads self_attn;
    float *w1_w, *w1_b, *w2_w, *w2_b;
    float *ln0_a, *ln0_b, *ln1_a, *ln1_b;
} capb200_tfm_enc_layer_grads;
typedef struct {
    capb200_mha_grads self_attn, src_attn;
    float *w1_w, *w1_b, *w2_w, *w2_b;
    float *ln0_a, *ln0_b, *ln1_a, *ln1_b, *ln2_a, *ln2_b;
} capb200_tfm_dec_layer_grads;
typedef struct {
    float *att_embed_w, *att_embed_b;
    capb200_tfm_enc_layer_grads enc[CAPB200_TFM_MAX_LAYERS];
    float *enc_norm_a, *enc_norm_b;
    capb200_tfm_dec_layer_grads dec[CAPB200_TFM_MAX_LAYERS];
    float *dec_norm_a, *dec_norm_b;
    float *lut, *pe;
    float *gen_w, *gen_b;
} capb200_tfm_grads;
typedef struct {
    int seq_per_img;
    unsigned long long seed;
    float label_smoothing, upstream, drop_prob_lm, dropout;
    const float* att_masks;        /* [B, R] or NULL */
    int keep_rows;                 /* drop_worst: > 0 keeps the `keep_rows` rows with the smallest loss (loss_wrapper.py:47-49, 75-77) */
    float* row_loss;               /* [N] or NULL */
} capb200_tfm_xe_opts;
typedef struct {
    int sample_n;
    float temperature;
    unsigned long long seed;
    float upstream;
    int baseline;                  /* CAPB200_BASELINE_GREEDY / CAPB200_BASELINE_LEAVE_ONE_OUT */
    float drop_prob_lm, dropout;
    const long long* forced_tokens;   /* [N, T] or NULL: replay these samples instead of drawing (tests) */
    const float* att_masks;
    int keep_rows;
    float* row_loss;
    const capb200_sampler_opts* sampler;            /* optional samplers, see capb200_scst_opts; NULL = multinomial + greedy baseline */
    const capb200_reward_weights* reward_weights;   /* optional reward weights, see capb200_scst_opts; NULL = CIDEr-D only */
} capb200_tfm_scst_opts;
int capb200_tfm_xe_step(capb200_tfm_engine* e, const float* att, int B, int R, const capb200_tfm_xe_opts* opts, const long long* labels, const float* masks,
                        int label_cols, const capb200_tfm_grads* grads, float* logprobs, float* loss, void* stream);
int capb200_tfm_scst_step(capb200_tfm_engine* e, const float* att, int B, int R, const capb200_tfm_scst_opts* opts, const capb200_cider_table* table,
                          const int* refs, const int* ref_offsets, int L, const capb200_tfm_grads* grads, long long* sample_seq, long long* greedy_seq,
                          float* sample_logprobs, float* reward, float* loss, void* stream);
/* gradient groups (see capb200_engine_set_grad_events), n <= 2: 0 generator + decoder + target embedding; 1 encoder + att_embed */
int capb200_tfm_set_grad_events(capb200_tfm_engine* e, void* const* events, int n);

/* ------------------------------------------------------------------------------------------------------------------
 * PPO fine-tuning (LossWrapper with opt.use_ppo, losses.py:267-357; loss_wrapper.py:39-53) of every family: one fused step of
 *   (1) the family's sampled forward in train mode, exactly as its *_scst_step draws it (opts: sample_n >= 2, temperature, seed, dropout
 *       rates, forced_tokens, att_masks, keep_rows / row_loss, sampler, reward_weights; baseline must be CAPB200_BASELINE_LEAVE_ONE_OUT);
 *   (2) the frozen old policy's teacher-forced pass over [0, seq[:, :-1]] on `old` -- an engine of the same family and configuration
 *       holding the old weights -- in eval mode, on `stream`; its log-probs lo [N, T, V+1] stay on `old`'s training tape;
 *   (3) the reward (cider * CIDEr-D + bleu * BLEU-4) and the leave-one-out advantage adv = s - mean of the image's other samples;
 *   (4) the criterion, mask[n, t] = 1 for t = 0 or seq[n, t-1] > 0, ratio = exp(lp[seq] - lo[seq]), eps = ppo->cliprange:
 *       pg = max(-adv ratio, -adv clamp(ratio, 1 - eps, 1 + eps)), kl = sum_v exp(lo_v) (lo_v - lp_v) over the full row,
 *       pg_loss / kl_loss / clipfrac = masked means of pg, kl and |ratio - 1| > eps,
 *       loss = pg_loss + kl_coef * kl_loss (reduction 'mean'), or with keep_rows > 0 the mean of the keep_rows smallest per-row masked
 *       means of pg + kl_coef * kl (drop_worst; row_loss receives every row's);
 *   (5) the backward through the new policy alone, into grads (every buffer OVERWRITTEN).
 * Outputs: sample_seq [N, T] int64, sample_logprobs [N, T, V+1], scores [N] (the rewarded scores in fp32, out['reward']), loss, pg_loss,
 * kl_loss, clipfrac [1].  The step runs eagerly (no CUDA graph); `old` must not be used by another call until it returns.
 * ---------------------------------------------------------------------------------------------------------------- */
typedef struct {
    float cliprange;           /* ppo_cliprange (0.2), > 0 */
    float kl_coef;             /* ppo_kl_coef (0.02), >= 0 */
} capb200_ppo_opts;
int capb200_updown_ppo_step(capb200_engine* e, capb200_engine* old, const float* fc, const float* att, int B, int R, const capb200_scst_opts* opts,
                            const capb200_ppo_opts* ppo, const capb200_cider_table* table, const int* refs, const int* ref_offsets, int L,
                            const capb200_updown_grads* grads, long long* sample_seq, float* sample_logprobs, float* scores, float* loss, float* pg_loss,
                            float* kl_loss, float* clipfrac, void* stream);
int capb200_att2in2_ppo_step(capb200_engine* e, capb200_engine* old, const float* fc, const float* att, int B, int R, const capb200_scst_opts* opts,
                             const capb200_ppo_opts* ppo, const capb200_cider_table* table, const int* refs, const int* ref_offsets, int L,
                             const capb200_att2in2_grads* grads, long long* sample_seq, float* sample_logprobs, float* scores, float* loss, float* pg_loss,
                             float* kl_loss, float* clipfrac, void* stream);
int capb200_newfc_ppo_step(capb200_engine* e, capb200_engine* old, const float* fc, const float* att, int B, int R, const capb200_scst_opts* opts,
                           const capb200_ppo_opts* ppo, const capb200_cider_table* table, const int* refs, const int* ref_offsets, int L,
                           const capb200_newfc_grads* grads, long long* sample_seq, float* sample_logprobs, float* scores, float* loss, float* pg_loss,
                           float* kl_loss, float* clipfrac, void* stream);
int capb200_aoa_ppo_step(capb200_aoa_engine* e, capb200_aoa_engine* old, const float* att, int B, int R, const capb200_aoa_scst_opts* opts,
                         const capb200_ppo_opts* ppo, const capb200_cider_table* table, const int* refs, const int* ref_offsets, int L,
                         const capb200_aoa_grads* grads, long long* sample_seq, float* sample_logprobs, float* scores, float* loss, float* pg_loss,
                         float* kl_loss, float* clipfrac, void* stream);
int capb200_tfm_ppo_step(capb200_tfm_engine* e, capb200_tfm_engine* old, const float* att, int B, int R, const capb200_tfm_scst_opts* opts,
                         const capb200_ppo_opts* ppo, const capb200_cider_table* table, const int* refs, const int* ref_offsets, int L,
                         const capb200_tfm_grads* grads, long long* sample_seq, float* sample_logprobs, float* scores, float* loss, float* pg_loss,
                         float* kl_loss, float* clipfrac, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Autograd entry points of every family: the forward of the fused training steps without their criterion, and the backward of a
 * caller-given dL/dlogprobs, so that any loss written in PyTorch trains an engine model (models.py: model.autograd).
 *   *_xe_vjp    teacher form: the forward of the family's xe_step over labels[..., :label_cols-1] (scheduled sampling included; the
 *               words fed land in opts->tokens_used), logprobs [N, label_cols-1, V+1] (caller zero-fills; columns >= steps stay zero).
 *   *_scst_vjp  sampling form: the sampler of the family's scst_step (multinomial at opts->temperature, the argmax with vjp->greedy, or
 *               the replay of opts->forced_tokens), sample_seq [N, T] and sample_logprobs [N, T, V+1]; rows already finished are zero.
 * The option structs are the fused steps' own: seed, dropout rates (0 = eval mode), att_masks, seq_per_img / sample_n, steps, ss_prob,
 * tokens_used and forced_tokens mean what they mean there; baseline, upstream, label_smoothing and reward_weights are not read, keep_rows
 * must be 0.  With vjp->forward_only nothing else runs and grads may be NULL.  Otherwise the same forward (same seed, same words: pass
 * the recorded tokens_used as labels with ss_prob = 0, or the drawn seq as forced_tokens) is followed by the backward of
 * dlogprobs [N, Tl, V+1] (Tl = label_cols-1 or T) through log_softmax and the model: d logits = G - exp(logprobs) * sum_v G per row, zero
 * for rows the forward did not produce.  Every grads buffer is OVERWRITTEN.  The calls run eagerly (no CUDA graph), record no
 * gradient-group events, and reuse the engine's training tape: one call at a time per engine.
 * ---------------------------------------------------------------------------------------------------------------- */
typedef struct {
    int forward_only;          /* 1: the forward alone */
    const float* dlogprobs;    /* [N, Tl, V+1] fp32 device, the upstream gradient of the backward (forward_only = 0) */
    int greedy;                /* sampling form: draw the argmax (sample_method 'greedy') instead of a multinomial sample */
} capb200_vjp_opts;
int capb200_updown_xe_vjp(capb200_engine* e, const float* fc, const float* att, int B, int R, const capb200_xe_opts* opts, const capb200_vjp_opts* vjp,
                          const long long* labels, int label_cols, const capb200_updown_grads* grads, float* logprobs, void* stream);
int capb200_updown_scst_vjp(capb200_engine* e, const float* fc, const float* att, int B, int R, const capb200_scst_opts* opts, const capb200_vjp_opts* vjp,
                            const capb200_updown_grads* grads, long long* sample_seq, float* sample_logprobs, void* stream);
int capb200_att2in2_xe_vjp(capb200_engine* e, const float* fc, const float* att, int B, int R, const capb200_xe_opts* opts, const capb200_vjp_opts* vjp,
                           const long long* labels, int label_cols, const capb200_att2in2_grads* grads, float* logprobs, void* stream);
int capb200_att2in2_scst_vjp(capb200_engine* e, const float* fc, const float* att, int B, int R, const capb200_scst_opts* opts, const capb200_vjp_opts* vjp,
                             const capb200_att2in2_grads* grads, long long* sample_seq, float* sample_logprobs, void* stream);
int capb200_newfc_xe_vjp(capb200_engine* e, const float* fc, const float* att, int B, int R, const capb200_xe_opts* opts, const capb200_vjp_opts* vjp,
                         const long long* labels, int label_cols, const capb200_newfc_grads* grads, float* logprobs, void* stream);
int capb200_newfc_scst_vjp(capb200_engine* e, const float* fc, const float* att, int B, int R, const capb200_scst_opts* opts, const capb200_vjp_opts* vjp,
                           const capb200_newfc_grads* grads, long long* sample_seq, float* sample_logprobs, void* stream);
int capb200_aoa_xe_vjp(capb200_aoa_engine* e, const float* att, int B, int R, const capb200_aoa_xe_opts* opts, const capb200_vjp_opts* vjp,
                       const long long* labels, int label_cols, const capb200_aoa_grads* grads, float* logprobs, void* stream);
int capb200_aoa_scst_vjp(capb200_aoa_engine* e, const float* att, int B, int R, const capb200_aoa_scst_opts* opts, const capb200_vjp_opts* vjp,
                         const capb200_aoa_grads* grads, long long* sample_seq, float* sample_logprobs, void* stream);
int capb200_tfm_xe_vjp(capb200_tfm_engine* e, const float* att, int B, int R, const capb200_tfm_xe_opts* opts, const capb200_vjp_opts* vjp,
                       const long long* labels, int label_cols, const capb200_tfm_grads* grads, float* logprobs, void* stream);
int capb200_tfm_scst_vjp(capb200_tfm_engine* e, const float* att, int B, int R, const capb200_tfm_scst_opts* opts, const capb200_vjp_opts* vjp,
                         const capb200_tfm_grads* grads, long long* sample_seq, float* sample_logprobs, void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Optimizer step of the training loop: utils.clip_gradient(optimizer, grad_clip_value) (captioning/utils/misc.py:156-160, called at
 * tools/train.py:193) + torch.optim.Adam.step() (built by build_optimizer, misc.py:186-205; tools/train.py:196) in ONE launch.
 *   table  [n_tensors][4] device pointers {param, grad, exp_avg, exp_avg_sq} (fp32, contiguous), itself in device memory
 *   numel  [n_tensors] element counts (device)
 *   chunks [n_chunks][2] int32 {tensor index, chunk index}; a chunk is capb200_adam_chunk_elems() elements (device)
 *   step   the 1-based step count AFTER this update (bias corrections 1 - beta^step);  clip_value <= 0 disables the clamp;
 *   write_clamped != 0 stores the clamped gradient back (clip_gradient's in-place side effect).  weight_decay is Adam's L2 term.
 * ---------------------------------------------------------------------------------------------------------------- */
int capb200_adam_chunk_elems(void);
int capb200_adam_step(const unsigned long long* table, const long long* numel, const int* chunks, int n_chunks, double lr, double beta1, double beta2,
                      double eps, double weight_decay, long step, double clip_value, int write_clamped, void* stream);


/* ------------------------------------------------------------------------------------------------------------------
 * Decode GEMM with any fused epilogue (tests and tools/gemm_trace.py): y = x[M,K] w[N,K]^T on fp32 device inputs, split into fp16 planes
 * in scratch memory, in mode CAPB200_MODE_TC_F16X3 or _TC_F16X1.  Every pointer in the epilogue is a device pointer; NULL turns an option
 * off.  Per element: + bias[col] + row_bias[row / rows_per_group, col] + gather_bias[gather_idx[row], col] + residual[row, col], then ReLU.
 * The kind follows from the fields: lstm != 0 is the fused nn.LSTMCell (N == 4H, gate-interleaved columns 4u+g, g in (i,f,g,o);
 * c_prev is read at row src_row[row], identity when src_row is NULL, zero state when src_row[row] < 0; writes c_out, h_f and, when h_hi
 * is set, the split planes h_hi / h_lo); otherwise C_hi != NULL stores the split planes C_hi / C_lo (fp16, as unsigned short) and C when
 * set; otherwise fp32 C.  Outputs must not overlap inputs.  Synchronous.
 * trace_host (or NULL): 296 x 16 %globaltimer stamps (ns) of one launch after three warm ones (tc_f16x3 only), one row per CTA: 0 set-up
 * done, 1 first operands landed, 2/3 main loop of the CTA's first / second tile done, 6/7 epilogue of tile 0 / 1 done, 8 kernel end.
 * ---------------------------------------------------------------------------------------------------------------- */
typedef struct {
    const float* bias;
    const float* row_bias;
    long ld_row_bias;
    int rows_per_group;
    const float* residual;
    long ld_res;
    int relu;
    float* C;
    long ldc;
    unsigned short* C_hi;
    unsigned short* C_lo;
    long ldcs;
    int lstm;
    int H;
    const float* c_prev;
    long ld_cprev;
    const int* src_row;
    float* c_out;
    long ld_cout;
    const float* gather_bias;
    long ld_gb;
    const int* gather_idx;
    float* h_f;
    unsigned short* h_hi;
    unsigned short* h_lo;
    long ld_h;
} capb200_gemm_epilogue;
int capb200_decode_gemm(const float* x, const float* w, int M, int N, int K, int mode, const capb200_gemm_epilogue* epi, unsigned long long* trace_host,
                        int n_slots, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* CAPB200_H_ */
