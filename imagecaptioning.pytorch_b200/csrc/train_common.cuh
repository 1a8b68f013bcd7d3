// The scaffold every fused training step shares (UpDown, Att2in2 and NewFC in engine.cu, AoANet in aoa_engine.cu, the Transformer in
// tfm_engine.cu): the tape buffers of the loss and the sampler, tape growth, the greedy baseline on the side stream, the word feed and the
// vocabulary step of the forward, the loss and its d logits, the option checks, and the eager-or-graph dispatch of the SCST step.  A family
// keeps its prologue, its core step, the backward through time and the weight gradients.
#pragma once
#include <cmath>
#include <cstring>
#include <functional>

#include "engine_common.cuh"

namespace capb200 {

// an fp32-only view (no fp16 planes) of a row-major activation
inline ActView f32_view(float* f, long ld) { return ActView{f, nullptr, nullptr, ld}; }

// The PPO criterion of a sampled step (run_ppo_step): its options, outputs, the scratch it keeps on the old policy's engine, and the old policy's
// teacher-forced pass old_pass(tokens_in [N, T], lo [N, T, V1], stream).
struct PpoArgs {
    float cliprange = 0.2f, kl_coef = 0.02f;
    float *scores = nullptr, *pg_loss = nullptr, *kl_loss = nullptr, *clipfrac = nullptr;
    long long* tokens_in = nullptr;
    float *lo = nullptr, *adv = nullptr;
    PpoScratch s{};
    std::function<int(const long long*, float*, cudaStream_t)> old_pass;
};

// One training step: SCST (sampled words, reward-weighted loss) or XE (teacher-forced words, cross-entropy).
struct TrainArgs {
    bool xe = false;
    int n = 1;                 // rows per image: train_sample_n (SCST) or seq_per_img (XE)
    int T = 0;                 // steps (positions) evaluated, and columns of the tape
    int Tl = 0;                // columns of the log-prob output [N, Tl, V1]
    float p = 0.f;             // the family's main dropout rate (drop_prob_lm; the Transformer's own `dropout`)
    float temperature = 1.f, upstream = 1.f, smoothing = 0.f;
    unsigned long long seed = 0;
    // SCST
    bool greedy_baseline = true;
    const capb200_cider_table* table = nullptr;
    const int* refs = nullptr; const int* ref_offsets = nullptr; int L = 0;     // CIDEr-D references; L = their length
    double w_cider = 1.0, w_bleu = 0.0;     // reward weights (capb200_reward_weights, by value)
    long long* sample_seq = nullptr; long long* greedy_seq = nullptr; float* reward = nullptr;
    const long long* forced = nullptr;      // replay these samples instead of drawing
    const float* mask = nullptr;            // [B, R] region mask or null
    float ss_prob = 0.f;                    // XE: scheduled sampling probability
    long long* tokens_used = nullptr;       // XE: optional [N, Tl] record of the words fed
    int keep = 0;                           // drop_worst: rows kept (0 = reduction 'mean')
    float* row_loss = nullptr;              // drop_worst: optional per-row loss output
    // XE
    const long long* labels = nullptr; long ld_labels = 0; const float* masks = nullptr; long ld_masks = 0;
    float* logprobs = nullptr; float* loss = nullptr;
    // the autograd entry points (capb200_*_vjp): stop after the forward, or replace the criterion by an outside dL/dlogprobs [N, Tl, V1]
    bool forward_only = false;
    const float* dlogprobs = nullptr;
    // SCST: how the samples are drawn -- the vocabulary step's select code (1 argmax, 2 multinomial, 4 top-k, 5 nucleus) and its k or p --
    // and how the eval-mode baseline is drawn (CAPB200_SAMPLE_*; forced_baseline [B, T] replays given captions instead)
    int select = 2;
    float top = 0.f;
    int baseline_method = CAPB200_SAMPLE_GREEDY;
    float baseline_top = 0.f;
    const long long* forced_baseline = nullptr;
    // PPO in place of RewardCriterion (leave-one-out advantage, no eval-mode baseline)
    const PpoArgs* ppo = nullptr;

    // The weighted reward runs only when it can differ from CIDEr-D alone: a BLEU weight <= 0 adds weight * 0.
    bool weighted_reward() const { return !xe && (w_bleu > 0.0 || w_cider != 1.0); }
    // kernels the weighted reward and a corpus table's build add to the CIDEr-D reward's two (scores, reward)
    int reward_extra_launches() const {
        const int build = table != nullptr && (!weighted_reward() || w_cider > 0.0) ? corpus_build_launches(table->t) : 0;
        return (weighted_reward() ? weighted_reward_launches(w_cider, w_bleu, true) - 2 : 0) + build;
    }
};

inline int vjp_train_args(const capb200_vjp_opts* v, TrainArgs* ta);

// A sampling method of capb200_sampler_opts -> the vocabulary step's select code, after checking its k or p.
inline int sampler_select(int method, float top, int* select) {
    CAPB_REQUIRE(method == CAPB200_SAMPLE_GREEDY || method == CAPB200_SAMPLE_MULTINOMIAL || method == CAPB200_SAMPLE_TOPK || method == CAPB200_SAMPLE_TOPP,
                 "unknown sampling method (greedy, multinomial, top-k or nucleus)");
    if (method == CAPB200_SAMPLE_TOPK) CAPB_REQUIRE(top >= 1.f && top <= 1e9f, "top-k sampling needs k >= 1");
    if (method == CAPB200_SAMPLE_TOPP) CAPB_REQUIRE(top > 0.f && top < 1.f, "nucleus sampling needs 0 < p < 1");
    *select = method == CAPB200_SAMPLE_GREEDY ? 1 : (method == CAPB200_SAMPLE_MULTINOMIAL ? 2 : method);
    return 0;
}

// Checks the SCST options every family shares and fills `ta`.  A family hands its own options over as capb200_scst_opts (drop_prob = its
// main dropout rate) and checks its other rates itself.  With `vjp` (an autograd entry point) no reward runs: the baseline is not read.
inline int scst_train_args(int B, const capb200_scst_opts& o, const capb200_cider_table* table, const int* refs, const int* ref_offsets, int L,
                           long long* sample_seq, long long* greedy_seq, float* sample_logprobs, float* reward, float* loss, int T, TrainArgs* ta,
                           const capb200_vjp_opts* vjp = nullptr) {
    const bool greedy_baseline = vjp == nullptr && o.baseline == CAPB200_BASELINE_GREEDY;
    if (vjp == nullptr) {
        CAPB_REQUIRE(greedy_baseline || o.baseline == CAPB200_BASELINE_LEAVE_ONE_OUT, "unknown baseline");
        CAPB_REQUIRE(!greedy_baseline || greedy_seq != nullptr, "the greedy baseline needs greedy_seq");
        CAPB_REQUIRE(greedy_baseline || o.sample_n >= 2, "the leave-one-out baseline needs sample_n >= 2");
    }
    CAPB_REQUIRE(o.sample_n >= 1 && o.sample_n <= 16 && B >= 1, "sample_n must be in 1..16");
    CAPB_REQUIRE(o.drop_prob >= 0.f && o.drop_prob < 1.f, "dropout rates must be in [0, 1)");
    CAPB_REQUIRE(o.temperature > 0.f, "temperature must be positive");
    CAPB_REQUIRE(o.keep_rows >= 0 && o.keep_rows <= B * o.sample_n, "keep_rows must be in 0..rows");
    if (o.sampler != nullptr) {
        const capb200_sampler_opts& s = *o.sampler;
        CAPB_REQUIRE(vjp == nullptr, "the autograd entry points draw through vjp->greedy or forced tokens, not a sampler struct");
        int baseline_select = 0;
        if (sampler_select(s.train_method, s.train_top, &ta->select) || sampler_select(s.baseline_method, s.baseline_top, &baseline_select)) return 1;
        CAPB_REQUIRE(greedy_baseline || (s.baseline_method == CAPB200_SAMPLE_GREEDY && s.forced_baseline == nullptr),
                     "a sampled or forced baseline needs CAPB200_BASELINE_GREEDY");
        ta->top = s.train_method == CAPB200_SAMPLE_TOPK || s.train_method == CAPB200_SAMPLE_TOPP ? s.train_top : 0.f;
        ta->baseline_method = s.baseline_method;
        ta->baseline_top = s.baseline_method == CAPB200_SAMPLE_TOPK || s.baseline_method == CAPB200_SAMPLE_TOPP ? s.baseline_top : 0.f;
        ta->forced_baseline = s.forced_baseline;
    }
    if (o.reward_weights != nullptr) {
        CAPB_REQUIRE(std::isfinite(o.reward_weights->cider) && std::isfinite(o.reward_weights->bleu), "reward weights must be finite");
        ta->w_cider = o.reward_weights->cider; ta->w_bleu = o.reward_weights->bleu;
    }
    ta->n = o.sample_n; ta->T = T; ta->Tl = T; ta->p = o.drop_prob; ta->temperature = o.temperature; ta->upstream = o.upstream;
    ta->seed = o.seed; ta->greedy_baseline = greedy_baseline; ta->table = table; ta->refs = refs; ta->ref_offsets = ref_offsets; ta->L = L;
    ta->sample_seq = sample_seq; ta->greedy_seq = greedy_seq; ta->reward = reward; ta->logprobs = sample_logprobs; ta->loss = loss;
    ta->forced = o.forced_tokens; ta->mask = o.att_masks; ta->keep = o.keep_rows; ta->row_loss = o.row_loss;
    return vjp != nullptr ? vjp_train_args(vjp, ta) : 0;
}

// Checks the XE options every family shares and fills `ta`; a family hands its own options over as capb200_xe_opts, as above.  T is the
// engine's seq_length.
inline int xe_train_args(int B, const capb200_xe_opts& o, const long long* labels, const float* masks, int label_cols, float* logprobs, float* loss,
                         int T, TrainArgs* ta, const capb200_vjp_opts* vjp = nullptr) {
    CAPB_REQUIRE(o.seq_per_img >= 1 && o.seq_per_img <= 16 && B >= 1, "seq_per_img must be in 1..16");
    CAPB_REQUIRE(o.drop_prob >= 0.f && o.drop_prob < 1.f, "dropout rates must be in [0, 1)");
    CAPB_REQUIRE(o.label_smoothing >= 0.f && o.label_smoothing < 1.f, "label_smoothing must be in [0, 1)");
    CAPB_REQUIRE(label_cols >= 2 && label_cols <= T + 2, "labels are [N, seq_length + 2] (BOS, words, EOS padding)");
    CAPB_REQUIRE(o.steps >= 1 && o.steps <= label_cols - 1, "steps must be in 1..label_cols-1");
    CAPB_REQUIRE(o.ss_prob >= 0.f && o.ss_prob <= 1.f, "ss_prob must be in [0, 1]");
    CAPB_REQUIRE(o.keep_rows >= 0 && o.keep_rows <= B * o.seq_per_img, "keep_rows must be in 0..rows");
    ta->xe = true;
    ta->n = o.seq_per_img; ta->T = o.steps; ta->Tl = label_cols - 1; ta->p = o.drop_prob; ta->upstream = o.upstream; ta->seed = o.seed;
    ta->smoothing = o.label_smoothing;
    ta->labels = labels; ta->ld_labels = label_cols; ta->masks = masks; ta->ld_masks = label_cols; ta->logprobs = logprobs; ta->loss = loss;
    ta->mask = o.att_masks; ta->ss_prob = o.ss_prob; ta->tokens_used = o.tokens_used; ta->keep = o.keep_rows; ta->row_loss = o.row_loss;
    return vjp != nullptr ? vjp_train_args(vjp, ta) : 0;
}

// The options of an autograd entry point: the forward alone (no criterion, no reward, no gradients), or the backward of an outside
// dL/dlogprobs.  Neither has a loss: drop_worst has no meaning there.
inline int vjp_train_args(const capb200_vjp_opts* v, TrainArgs* ta) {
    CAPB_REQUIRE(v->forward_only || v->dlogprobs != nullptr, "the backward needs dlogprobs");
    CAPB_REQUIRE(ta->keep == 0, "keep_rows belongs to the fused steps' criterion");
    CAPB_REQUIRE(ta->xe || !v->greedy || ta->forced == nullptr, "greedy draws and forced tokens exclude each other");
    ta->forward_only = v->forward_only != 0;
    ta->dlogprobs = ta->forward_only ? nullptr : v->dlogprobs;
    if (v->greedy) ta->select = 1;
    ta->greedy_baseline = false;
    return 0;
}

// The buffers every training tape has: d loss / d logits, the criterion's scratch, the greedy baseline's log-probs, the split-K scratch of
// the skinny GEMMs, and the sampling loop's own word state (the greedy baseline runs concurrently on the decode workspace).  Each family's
// tape derives from it, so the helpers below take a StepTape&.
struct StepTape {
    float* DL;                                 // [N, T, V1]
    float *mask_sum, *item_loss, *glp, *skinny;
    size_t skinny_floats;
    double* scores;                            // [N + B] hypothesis scores, then [N + B] BLEU-4 of the weighted reward
    int *s_tokens, *s_unfinished, *s_forced;
    float *row_loss, *row_msum, *row_coef;     // drop_worst: per-row loss, mask count and gradient coefficient

    // TN = rows of the tape (positions x N); glp_floats = the greedy baseline's log-prob buffer
    void layout(Arena& a, int B, int N, long TN, int V1, long glp_floats) {
        DL = a.take<float>(TN * V1);
        mask_sum = a.take<float>(8);
        item_loss = a.take<float>(TN);
        glp = a.take<float>(glp_floats);
        skinny_floats = (size_t)4 << 20;       // split-K partial sums (16 MB)
        skinny = a.take<float>((long)skinny_floats);
        scores = a.take<double>(2 * ((long)N + B));
        s_tokens = a.take<int>(N); s_unfinished = a.take<int>(N); s_forced = a.take<int>(N);
        row_loss = a.take<float>(N); row_msum = a.take<float>(N); row_coef = a.take<float>(N);
    }
};

// Lays `tp` out on the engine's training tape (`layout(tp, arena)`), growing the tape first if the layout does not fit; growing synchronises.
template <class Tape, class Layout>
int carve_tape(char** tape, size_t* tape_bytes, Tape& tp, cudaStream_t st, Layout layout) {
    Arena dry;
    Tape sized;
    layout(sized, dry);
    if (grow_buffer(reinterpret_cast<void**>(tape), tape_bytes, dry.off + 256, st)) return 1;
    Arena ar;
    ar.base = *tape;
    layout(tp, ar);
    return 0;
}

// The skinny-GEMM runner of a training step on the tape's split-K scratch: wgmma 3xTF32 GEMMs through the engine's tf32 context unless
// the engine is in simt_fp32 mode.  Each step starts a new context step: the weights may have changed since the last one.
inline Skinny step_gemms(Tf32Context** ctx, bool tc, const StepTape& tp, cudaStream_t st) {
    if (tc && *ctx == nullptr) *ctx = tf32_context_create();
    tf32_context_new_step(*ctx);
    Skinny sk{tp.skinny, tp.skinny_floats, tc ? 1 : 0, st};
    sk.ctx = *ctx;
    return sk;
}

// The eval-mode baseline of an SCST step: the regular decode on B rows, without dropout -- greedy, or drawn as sc_sample_method says from the
// step's seed XOR kBaselineSalt (an XOR, so that the salt of a graph replay carries over: dropout.cuh), or the replay of given captions.  It and the train-mode sampling
// forward are independent chains of small, latency-bound kernels, so the baseline runs on the engine's side stream -- forked from the step's
// stream, joined before the reward -- unless the side stream or its events cannot be created.  Three calls: fork at
// the top of the step, enqueue where the family wants its launches issued, join (inside loss_backward).
struct StepBaseline {
    static constexpr unsigned long long kBaselineSalt = 0x5bd1e9955bd1e995ull;
    bool needed = false;
    cudaStream_t st = nullptr;      // where its launches go
    cudaEvent_t done = nullptr;     // recorded on the side stream after them; null when they run on the step's stream
    int method = CAPB200_SAMPLE_GREEDY;
    float top = 0.f;
    unsigned long long seed = 0;
    const long long* forced = nullptr;

    int fork(const TrainArgs& ta, cudaStream_t* side, cudaEvent_t* ev_fork, cudaEvent_t* ev_join, cudaStream_t step_st) {
        needed = !ta.xe && ta.greedy_baseline;
        forced = ta.forced_baseline;
        method = forced != nullptr ? CAPB200_SAMPLE_FORCED : ta.baseline_method;
        top = ta.baseline_top;
        seed = method == CAPB200_SAMPLE_GREEDY || method == CAPB200_SAMPLE_FORCED ? 0ull : ta.seed ^ kBaselineSalt;
        st = step_st;
        done = nullptr;
        if (!needed) return 0;
        bool ok = *side != nullptr || create_side_stream(side) == cudaSuccess;
        if (ok && *ev_fork == nullptr) ok = cudaEventCreateWithFlags(ev_fork, cudaEventDisableTiming) == cudaSuccess;
        if (ok && *ev_join == nullptr) ok = cudaEventCreateWithFlags(ev_join, cudaEventDisableTiming) == cudaSuccess;
        if (!ok) { (void)cudaGetLastError(); return 0; }
        CAPB_CHECK_CUDA(cudaEventRecord(*ev_fork, step_st));
        CAPB_CHECK_CUDA(cudaStreamWaitEvent(*side, *ev_fork, 0));
        st = *side;
        done = *ev_join;
        return 0;
    }
    // decode(opts, tokens_in, greedy_seq, logprobs, stream) is the family's capb200_*decode_sample (tokens_in [B, T]: the forced captions or null)
    template <class Decode>
    int enqueue(int B, int T, int V1, long long* greedy_seq, float* glp, Decode decode) const {
        if (!needed) return 0;
        CAPB_NVTX("capb200 scst: baseline (eval mode, side stream)");
        capb200_sample_opts so;
        memset(&so, 0, sizeof(so));
        so.edits.unk_col = -1; so.sample_n = 1; so.method = method; so.temperature = 1.f; so.seed = seed; so.steps = T; so.top = top;
        CAPB_CHECK_CUDA(cudaMemsetAsync(glp, 0, sizeof(float) * (size_t)B * T * V1, st));
        CAPB_CHECK_CUDA(cudaMemsetAsync(greedy_seq, 0, sizeof(long long) * (size_t)B * T, st));
        if (decode(&so, forced, greedy_seq, glp, static_cast<void*>(st))) return 1;
        if (done != nullptr) CAPB_CHECK_CUDA(cudaEventRecord(done, st));
        return 0;
    }
    int join(cudaStream_t step_st) const {
        if (done != nullptr) CAPB_CHECK_CUDA(cudaStreamWaitEvent(step_st, done, 0));
        return 0;
    }
};

// The words fed at step t into `tok` (the tape's column t).  XE feeds the labels -- or, with scheduled sampling, draws from the model's
// previous prediction (AttModel.py:145-154) -- and records them in ta.tokens_used if asked; SCST feeds the previous step's draw.
inline int feed_tokens(const TrainArgs& ta, const StepTape& tp, int N, int V1, int t, int* tok, cudaStream_t st) {
    if (!ta.xe) {
        CAPB_CHECK_CUDA(cudaMemcpyAsync(tok, tp.s_tokens, sizeof(int) * N, cudaMemcpyDeviceToDevice, st));
        return 0;
    }
    if (t >= 1 && ta.ss_prob > 0.f) {
        if (ss_select_launch(N, V1, ta.logprobs + (long)(t - 1) * V1, (long)ta.Tl * V1, ta.labels, ta.ld_labels, t, ta.seed, ta.ss_prob, tok, st)) return 1;
    } else if (load_token_column_launch(ta.labels, ta.ld_labels, t, N, tok, st)) return 1;
    if (ta.tokens_used != nullptr && store_token_column_launch(tok, N, ta.tokens_used, ta.Tl, t, st)) return 1;
    return 0;
}

// The vocabulary step at step t: log_softmax of the logits at ta.logprobs[:, t] in place; SCST also draws the next words (ta.select at
// ta.temperature, or the replay of ta.forced) into tp.s_tokens and ta.sample_seq.  The full log-softmax row stays in ta.logprobs whatever
// the sampler keeps: it is what the criterion and the gradient read (AttModel.py:337,347).
inline int train_vocab_step(const TrainArgs& ta, const StepTape& tp, int N, int V1, int t, cudaStream_t st) {
    VocabStepArgs va;
    va.rows = N; va.V1 = V1; va.logits = ta.logprobs + (long)t * V1; va.ld = (long)ta.Tl * V1;
    if (!ta.xe) {
        va.select = ta.select; va.top = ta.top; va.temperature = ta.temperature; va.seed = ta.seed; va.step = (unsigned long long)t;
        va.unfinished = tp.s_unfinished; va.first_step = (t == 0); va.tokens_out = tp.s_tokens;
        va.seq_out = ta.sample_seq; va.ld_seq = ta.T; va.t = t;
        if (ta.forced != nullptr) {
            if (load_token_column_launch(ta.forced, ta.T, t, N, tp.s_forced, st)) return 1;
            va.select = 3; va.forced = tp.s_forced;
        }
    }
    return vocab_step_launch(va, st);
}

// PPO's loss and d loss / d logits into tp.DL: the old policy's teacher-forced pass over [0, seq[:, :-1]], the reward with the leave-one-out
// advantage (losses.py:300-306), then the clipped-ratio + KL criterion.
inline int ppo_loss_backward(const TrainArgs& ta, const StepTape& tp, int B, int N, int V1, cudaStream_t st) {
    const PpoArgs& pa = *ta.ppo;
    const int T = ta.T;
    if (ppo_shift_launch(ta.sample_seq, N, T, pa.tokens_in, st) || pa.old_pass(pa.tokens_in, pa.lo, st)) return 1;
    if (!ta.weighted_reward()) {
        if (cider_reward_launch(ta.table->t, ta.sample_seq, N, nullptr, B, T, ta.refs, ta.ref_offsets, ta.L, tp.scores, pa.adv, 1, 1, st)) return 1;
    } else if (weighted_reward_launch(ta.table ? ta.table->t : nullptr, ta.w_cider, ta.w_bleu, ta.sample_seq, N, nullptr, B, T, ta.refs, ta.ref_offsets, ta.L,
                                      tp.scores, tp.scores + N + B, pa.adv, 1, 1, st)) return 1;
    return ppo_loss_backward_launch(ta.logprobs, (long)ta.Tl * V1, pa.lo, ta.sample_seq, pa.adv, tp.scores, N, T, V1, pa.cliprange, pa.kl_coef, ta.upstream,
                                    ta.keep, pa.s, tp.DL, pa.scores, ta.loss, ta.row_loss ? ta.row_loss : tp.row_loss, pa.pg_loss, pa.kl_loss, pa.clipfrac, st);
}

// The loss and d loss / d logits into tp.DL: the XE criterion (LanguageModelCriterion / LabelSmoothing), or -- after joining the greedy
// baseline -- the reward (CIDEr-D, or the weighted CIDEr-D + BLEU-4), RewardCriterion, drop_worst and the d logits of the SCST loss.
inline int loss_backward(const TrainArgs& ta, const StepTape& tp, const StepBaseline& gb, int B, int N, int V1, cudaStream_t st) {
    const int T = ta.T;
    const long ld_lp = (long)ta.Tl * V1;
    float* row_loss = ta.row_loss ? ta.row_loss : tp.row_loss;
    if (ta.dlogprobs != nullptr)
        return logsoftmax_vjp_launch(ta.logprobs, ta.dlogprobs, ld_lp, ta.xe ? nullptr : ta.sample_seq, N, T, V1, tp.DL, st);
    if (ta.xe)
        return xe_loss_backward_launch(ta.logprobs, ld_lp, ta.labels, ta.ld_labels, ta.masks, ta.ld_masks, N, T, ta.Tl, V1, ta.smoothing, ta.upstream,
                                       tp.mask_sum, tp.item_loss, tp.DL, ta.loss, st, ta.keep, row_loss, tp.row_msum, tp.row_coef);
    if (ta.ppo != nullptr) return ppo_loss_backward(ta, tp, B, N, V1, st);
    if (gb.join(st)) return 1;     // the reward needs the baseline captions
    const long long* greedy = ta.greedy_baseline ? ta.greedy_seq : nullptr;
    if (!ta.weighted_reward()) {
        if (cider_reward_launch(ta.table->t, ta.sample_seq, N, greedy, B, T, ta.refs, ta.ref_offsets, ta.L, tp.scores, ta.reward, T, T, st)) return 1;
    } else if (weighted_reward_launch(ta.table ? ta.table->t : nullptr, ta.w_cider, ta.w_bleu, ta.sample_seq, N, greedy, B, T, ta.refs, ta.ref_offsets, ta.L,
                                      tp.scores, tp.scores + N + B, ta.reward, T, T, st)) return 1;
    float* rl = ta.keep > 0 ? row_loss : nullptr;
    if (reward_criterion_fwd_launch(ta.logprobs, ld_lp, V1, ta.sample_seq, ta.reward, N, T, ta.loss, rl, tp.mask_sum, st)) return 1;
    if (ta.keep > 0 && scst_drop_worst_launch(ta.sample_seq, rl, N, T, ta.keep, ta.upstream, tp.row_msum, tp.row_coef, ta.loss, st)) return 1;
    return scst_dlogits_launch(ta.logprobs, ld_lp, ta.sample_seq, ta.reward, tp.mask_sum, ta.upstream, N, T, V1, tp.DL, st, ta.keep > 0 ? tp.row_coef : nullptr);
}

// ---- the logit head in the training steps (logit_layers = k > 1, AttModel.py:87-92) -------------------------------------------------------
// Hidden layer i's dropout masks are keyed by (the step's seed, site kHeadDropSite + i, position t), replayable with capb200_dropout_mask.
constexpr unsigned kHeadDropSite = 200;

// The head's training tape for TN = T * N rows: the k - 1 post-dropout activations [N, T, H] (slot i = layer i), then two gradient slabs.
inline int head_train_tape(EngineBase* e, long TN, cudaStream_t st) {
    if (e->logit_layers == 1) return 0;
    const size_t need = sizeof(float) * (size_t)(e->logit_layers + 1) * TN * e->head_H;
    return grow_buffer(reinterpret_cast<void**>(&e->head_tape), &e->head_tape_bytes, need, st);
}
inline float* head_slot(EngineBase* e, long TN, int i) { return e->head_tape + (size_t)i * TN * e->head_H; }

// Step t of the forward: x [N, H] (pitch ld) is the core's output; hidden layer i writes y_i = dropout(relu(x W_i^T + b_i)) into row (n, t)
// of its tape slot.  *in / *ld_in: what the vocabulary Linear reads (x itself when k = 1).
inline int head_train_forward(EngineBase* e, const Skinny& sk, const float* x, long ld, int N, int T, int t, unsigned long long seed, const float** in,
                              long* ld_in, cudaStream_t st) {
    const int H = e->head_H;
    const long TN = (long)T * N;
    for (int i = 0; i + 1 < e->logit_layers; ++i) {
        float* y = head_slot(e, TN, i) + (long)t * H;
        if (sk.lin(x, ld, e->head_w[i], H, e->head_b[i], y, (long)T * H, N, H, H, 0)) return 1;
        if (relu_dropout_apply_launch(y, N, H, (long)T * H, seed, kHeadDropSite + i, (unsigned)t, e->head_drop, st)) return 1;
        e->launches += 2;
        x = y;
        ld = (long)T * H;
    }
    *in = x;
    *ld_in = ld;
    return 0;
}

// loss_backward, then the backward of the output head batched over all (n, t) -- it is not recurrent: the vocabulary Linear [V1, H] (its
// input is the last hidden activation, or `out` [N, T, H] -- the core's output -- when k = 1), then the hidden layers from the last to the
// first (mask * relu', weight and bias gradients, input gradient), so that dOUT [N, T, H] ends up holding d loss / d core output.  All of it
// is gradient group 0, whose event `ev` is recorded here.
inline int loss_and_logit_backward(EngineBase* e, const TrainArgs& ta, const StepTape& tp, const StepBaseline& gb, const Skinny& sk, int B, int N, int V1,
                                   int H, const float* logit_w, const float* out, float* dOUT, float* g_logit_w, float* g_logit_b, cudaEvent_t ev,
                                   cudaStream_t st) {
    const int TN = ta.T * N;
    const int L = e->logit_layers - 1;
    if (loss_backward(ta, tp, gb, B, N, V1, st)) return 1;
    float* dy = L ? head_slot(e, TN, L) : dOUT;           // d loss / d (the vocabulary Linear's input)
    float* dz = L ? head_slot(e, TN, L + 1) : nullptr;
    if (sk.dgrad(TN, H, V1, tp.DL, V1, logit_w, H, dy, H, 0)) return 1;            // dY = DL * W
    if (sk.wgrad(V1, H, TN, tp.DL, V1, L ? head_slot(e, TN, L - 1) : out, H, g_logit_w, H, 0)) return 1;     // dW = DL^T * Y
    if (colsum_launch(TN, V1, tp.DL, V1, g_logit_b, 0, st)) return 1;
    const float scale = 1.f / (1.f - e->head_drop);
    for (int i = L - 1; i >= 0; --i) {
        const float* y = head_slot(e, TN, i);
        const float* x = i ? head_slot(e, TN, i - 1) : out;
        if (relu_dropout_backward_launch((long)TN * H, y, dy, dz, scale, st)) return 1;                    // y > 0 iff kept and relu' = 1
        if (sk.wgrad(H, H, TN, dz, H, x, H, e->head_gw[i], H, 0)) return 1;
        if (colsum_launch(TN, H, dz, H, e->head_gb[i], 0, st)) return 1;
        if (sk.dgrad(TN, H, H, dz, H, e->head_w[i], H, i ? dy : dOUT, H, 0)) return 1;
        e->launches += 4;
    }
    return record_group_event(ev, st);
}

// q | k | v weight and bias gradients of a self-attention block from d_qkv [rows, 3D] and its input x [rows, D]: one GEMM / one column
// reduction when the caller laid the three tensors out back to back (the Python mirror's flat gradient buffer does), else three.  The column
// reductions it launches are added to *colsums when that is given.
template <class Grads>
int qkv_grads(const Skinny& sk, int rows, int D, const float* d_qkv, const float* x, const Grads& g, long* colsums, cudaStream_t st) {
    int rc = 0;
    if (g.k_w == g.q_w + (long)D * D && g.v_w == g.k_w + (long)D * D) {
        rc |= sk.wgrad(3 * D, D, rows, d_qkv, 3 * D, x, D, g.q_w, D, 0);
    } else {
        rc |= sk.wgrad(D, D, rows, d_qkv, 3 * D, x, D, g.q_w, D, 0);
        rc |= sk.wgrad(D, D, rows, d_qkv + D, 3 * D, x, D, g.k_w, D, 0);
        rc |= sk.wgrad(D, D, rows, d_qkv + 2 * D, 3 * D, x, D, g.v_w, D, 0);
    }
    const bool packed_b = g.k_b == g.q_b + D && g.v_b == g.k_b + D;
    if (packed_b) {
        rc |= colsum_launch(rows, 3 * D, d_qkv, 3 * D, g.q_b, 0, st);
    } else {
        rc |= colsum_launch(rows, D, d_qkv, 3 * D, g.q_b, 0, st);
        rc |= colsum_launch(rows, D, d_qkv + D, 3 * D, g.k_b, 0, st);
        rc |= colsum_launch(rows, D, d_qkv + 2 * D, 3 * D, g.v_b, 0, st);
    }
    if (colsums != nullptr) *colsums += packed_b ? 1 : 3;
    return rc;
}

// An eager training step: the seed arguments are the effective seeds (a graph replay of an SCST step may have left a salt behind).
template <class Step>
int run_eager_step(cudaStream_t st, Step step) {
    if (dropout_salt_set_all(0ull, st)) return 1;
    return step();
}

// A step of an autograd entry point (capb200_*_vjp): eager, and with the engine's gradient-group events unset -- its gradients go to the
// caller's own table, which no data-parallel listener waits on.
template <class Step>
int run_vjp_step(EngineBase* e, cudaStream_t st, Step step) {
    cudaEvent_t saved[EngineBase::kMaxGradGroups];
    for (int i = 0; i < e->grad_groups; ++i) { saved[i] = e->grad_events[i]; e->grad_events[i] = nullptr; }
    const int rc = run_eager_step(st, step);
    for (int i = 0; i < e->grad_groups; ++i) e->grad_events[i] = saved[i];
    return rc;
}

// Runs one SCST step, `step(fc, att, ta, stream)`, as ONE CUDA graph.  Its ~900-4900 kernels are 5-30 us each, every launch boundary costs
// ~2 us on the stream, the host needs milliseconds to enqueue them, and nothing about the sequence depends on data: the step is captured the
// second time a configuration is seen and replayed afterwards with a fresh seed (dropout.cuh: seed salt).  The features fc / att and the
// region mask ta.mask are copied into the engine-owned staging buffer first, so that the graph reads stable addresses (an input of zero
// bytes is not staged and reaches the step as null); the key covers every option but the seed (the samplers and the reward weights by value), the gradient and
// weight tables, every pointer the step touches and the shapes.  The gradient-group events a data-parallel caller listens to become external event-record nodes of the
// graph (record_group_event) and are part of the key.  The step stays eager with CAPB200_SCST_GRAPH=0, in the simt_fp32 mode, when forced
// samples or baseline captions are replayed, and once a capture has failed.
template <class Engine, class Opts, class Grads, class Args, class Step>
int run_scst_step(Engine* e, const Opts* opts, const Grads* grads, const Args& ta, const float* fc, size_t fc_bytes, const float* att, size_t att_bytes,
                  int B, int R, cudaStream_t st, Step step) {
    // the weighted reward's kernels are counted here, so that the families' hand-kept counts stay those of the CIDEr-D reward
    auto counted = [&](const float* f, const float* a, const Args& t, cudaStream_t s) {
        const int rc = step(f, a, t, s);
        e->launches += t.reward_extra_launches();
        return rc;
    };
    if (!StepGraph::enabled() || !e->tc || ta.forced != nullptr || ta.forced_baseline != nullptr || e->sg.broken)
        return run_eager_step(st, [&] { return counted(fc, att, ta, st); });
    cudaStream_t gst = e->sg.enter(st);             // a capturable engine-owned stream, ordered after the caller's stream
    const void* srcs[3] = {fc, att, ta.mask};
    const size_t bytes[3] = {fc_bytes, att_bytes, ta.mask ? sizeof(float) * (size_t)B * R : 0};
    size_t off[3];
    if (e->sg.stage_inputs(3, srcs, bytes, off, gst)) return 1;
    auto staged = [&](int i) { return bytes[i] ? reinterpret_cast<const float*>(e->sg.stage + off[i]) : nullptr; };
    Args ts = ta;
    ts.mask = staged(2);
    unsigned long long key = 1469598103934665603ull;
    Opts o2 = *opts; o2.seed = 0; o2.att_masks = ts.mask; o2.sampler = nullptr; o2.reward_weights = nullptr;
    StepGraph::mix(key, &o2, sizeof(o2));
    const double weights[2] = {ta.w_cider, ta.w_bleu};      // the values: the caller's structs may keep their addresses while they change
    StepGraph::mix(key, weights, sizeof(weights));
    const int methods[2] = {ta.select, ta.baseline_method};
    const float tops[2] = {ta.top, ta.baseline_top};
    unsigned long long table_key[3];                          // a corpus table's slots move when it grows; the kind decides the build
    cider_table_key(ta.table ? ta.table->t : nullptr, table_key);
    StepGraph::mix(key, methods, sizeof(methods)); StepGraph::mix(key, tops, sizeof(tops)); StepGraph::mix(key, table_key, sizeof(table_key)); StepGraph::mix(key, grads, sizeof(*grads)); StepGraph::mix(key, &e->w, sizeof(e->w));
    const void* ptrs[] = {ta.table, ta.refs, ta.ref_offsets, ta.sample_seq, ta.greedy_seq, ta.logprobs, ta.reward, ta.loss, e->tape, e->ws, e->wblock, e->sg.stage, gst};
    StepGraph::mix(key, ptrs, sizeof(ptrs));
    StepGraph::mix(key, e->grad_events, sizeof(cudaEvent_t) * e->grad_groups);
    if (e->logit_layers > 1) {                                // the logit head's weights, gradient buffers, dropout rate and tape
        const size_t n = sizeof(void*) * (e->logit_layers - 1);
        StepGraph::mix(key, e->head_w.data(), n); StepGraph::mix(key, e->head_b.data(), n);
        StepGraph::mix(key, e->head_gw.data(), n); StepGraph::mix(key, e->head_gb.data(), n);
        const void* hp[2] = {e->head_tape, e->head_block};
        StepGraph::mix(key, hp, sizeof(hp)); StepGraph::mix(key, &e->head_drop, sizeof(float)); StepGraph::mix(key, &e->logit_layers, sizeof(int));
    }
    const int dims[] = {B, R, ta.L};
    StepGraph::mix(key, dims, sizeof(dims));
    const int rc = run_step_graph(e->sg, key, opts->seed, &e->launches, gst, [&]() { return counted(staged(0), staged(1), ts, gst); });
    if (e->sg.leave(st, gst)) return 1;
    return rc;
}

// Runs one PPO step eagerly: `step()` is the family's sampled training step with ta.ppo set.  The old policy `old` is an engine of the same
// family and configuration whose weights stay frozen; its teacher-forced pass, old_pass(opts, tokens_in, lo, stream) -- the family's
// capb200_*decode_sample on `old` -- runs in eval mode on the step's stream, and the criterion's scratch (lo [N, T, V1], the shifted words, the
// advantage and the per-position terms) lives on the old engine's training tape, which nothing else uses while it does not train.
template <class Engine, class Args, class OldPass, class Step>
int run_ppo_step(Engine* e, Engine* old, const capb200_ppo_opts* po, Args& ta, int B, float* scores, float* pg_loss, float* kl_loss, float* clipfrac,
                 cudaStream_t st, OldPass old_pass, Step step) {
    CAPB_REQUIRE(po && old && scores && pg_loss && kl_loss && clipfrac, "null argument");
    if (check_ready(old)) return 1;
    CAPB_REQUIRE(old != e, "the old policy needs an engine of its own");
    CAPB_REQUIRE(memcmp(&old->cfg, &e->cfg, sizeof(e->cfg)) == 0 && old->logit_layers == e->logit_layers,
                 "the old policy's engine must have the family and configuration of the new one");
    CAPB_REQUIRE(!ta.greedy_baseline, "PPO takes the leave-one-out advantage: baseline must be CAPB200_BASELINE_LEAVE_ONE_OUT");
    CAPB_REQUIRE(std::isfinite(po->cliprange) && po->cliprange > 0.f && std::isfinite(po->kl_coef) && po->kl_coef >= 0.f,
                 "PPO needs cliprange > 0 and kl_coef >= 0");
    const int n = ta.n, N = B * n, T = ta.T;
    const size_t NT = (size_t)N * T;
    PpoArgs pa;
    pa.cliprange = po->cliprange; pa.kl_coef = po->kl_coef;
    pa.scores = scores; pa.pg_loss = pg_loss; pa.kl_loss = kl_loss; pa.clipfrac = clipfrac;
    auto layout = [&](Arena& a) {
        pa.lo = a.take<float>(NT * e->V1);
        pa.tokens_in = a.take<long long>(NT);
        pa.adv = a.take<float>(N);
        pa.s.terms = a.take<float>(3 * NT);
        pa.s.row_msum = a.take<float>(N); pa.s.row_coef = a.take<float>(N); pa.s.mask_sum = a.take<float>(1);
    };
    Arena dry;
    layout(dry);
    if (grow_buffer(reinterpret_cast<void**>(&old->tape), &old->tape_bytes, dry.off + 256, st)) return 1;
    Arena ar;
    ar.base = old->tape;
    layout(ar);
    capb200_sample_opts so;
    memset(&so, 0, sizeof(so));
    so.edits.unk_col = -1; so.sample_n = n; so.method = CAPB200_SAMPLE_TEACHER; so.temperature = 1.f; so.steps = T;
    pa.old_pass = [&](const long long* tok, float* lo, cudaStream_t s) { return old_pass(&so, tok, lo, static_cast<void*>(s)); };
    ta.ppo = &pa;
    // the launches PPO adds to the sampled step's count: the word shift, and the criterion's three against RewardCriterion's two
    return run_eager_step(st, [&] {
        const int rc = step();
        e->launches += ta.reward_extra_launches() + 2;
        return rc;
    });
}

}  // namespace capb200
