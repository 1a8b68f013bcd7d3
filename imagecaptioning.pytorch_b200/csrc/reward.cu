// SCST reward on the device: CIDEr-D over token ids, self-critical baseline, and RewardCriterion forward / backward.
//
// Replaces the host-side Python path the reference takes every SCST step:
//   get_self_critical_reward   captioning/utils/rewards.py:41-81   (.cpu().numpy(), str() of every id, dict loops)
//   CiderD.compute_score       cider/pyciderevalcap/ciderD/ciderD.py:31-56 -> ciderD_scorer.py:17-32,53-79,156-208
//   RewardCriterion.forward    captioning/modules/losses.py:22-37
// Arithmetic follows the reference exactly, in float64 like numpy:
//   * a caption is its tokens up to and INCLUDING the first 0 (array_to_str keeps "0"),
//   * tf-idf weight of an n-gram = tf * (log(ref_len) - log(max(1, df))), df from the preprocessed table,
//   * per order n: sum over the hypothesis' distinct n-grams of min(w_h, w_r) * w_r, divided by |h||r| when both are
//     non-zero, times exp(-(len_h - len_r)^2 / (2 * 6^2)) where len counts BIGRAMS (ciderD_scorer.py:177-178),
//   * score = 10 * mean over references of the mean over n = 1..4.
//
// The BLEU-4 term of the reward (rewards.py:68-74, coco-caption/pycocoevalcap/bleu) and the weighted sum of the two terms are here too.
#include <cmath>
#include <vector>

#include "../../include/capb200.h"
#include "common.cuh"
#include "cider_table.cuh"
#include "kernels.cuh"

namespace capb200 {

static_assert(CIDER_MAXL_LONG == CAPB200_MAX_SEQ_LENGTH, "the rewards' long form holds the longest caption the engines produce");

CiderTable* cider_table_create(const int* keys, const double* df, long n, double ref_len, cudaStream_t stream) {
    unsigned long long cap = 64;
    while (cap < (unsigned long long)(2 * n + 1)) cap <<= 1;
    std::vector<CiderSlot> host(cap);
    for (auto& s : host) { s.key[0] = -2; s.key[1] = s.key[2] = s.key[3] = -2; s.idf = 0.0; }
    const double log_ref = log(ref_len);
    for (long i = 0; i < n; ++i) {
        const int* k = keys + 4 * i;
        unsigned long long h = cider_hash(k[0], k[1], k[2], k[3]) & (cap - 1);
        while (host[h].key[0] != -2) {
            if (host[h].key[0] == k[0] && host[h].key[1] == k[1] && host[h].key[2] == k[2] && host[h].key[3] == k[3]) break;
            h = (h + 1) & (cap - 1);
        }
        host[h].key[0] = k[0]; host[h].key[1] = k[1]; host[h].key[2] = k[2]; host[h].key[3] = k[3];
        host[h].idf = log_ref - log(df[i] > 1.0 ? df[i] : 1.0);
    }
    CiderTable* t = new CiderTable();
    t->mask = cap - 1;
    t->log_ref_len = log_ref;
    t->entries = n;
    if (cudaMalloc(&t->slots, cap * sizeof(CiderSlot)) != cudaSuccess) {
        set_error("cider_table_create: cudaMalloc failed");
        delete t;
        return nullptr;
    }
    if (cudaMemcpyAsync(t->slots, host.data(), cap * sizeof(CiderSlot), cudaMemcpyHostToDevice, stream) != cudaSuccess ||
        cudaStreamSynchronize(stream) != cudaSuccess) {
        set_error("cider_table_create: upload failed");
        cudaFree(t->slots);
        delete t;
        return nullptr;
    }
    return t;
}

void cider_table_destroy(CiderTable* t) {
    if (t == nullptr) return;
    cudaFree(t->slots);
    if (t->used) cudaFree(t->used);
    delete t;
}

CiderTable* cider_corpus_table_create() {
    CiderTable* t = new CiderTable();
    t->corpus = true;
    if (cudaMalloc(&t->used, sizeof(unsigned int)) != cudaSuccess) {
        (void)cudaGetLastError();
        set_error("cider_corpus_table_create: cudaMalloc failed");
        delete t;
        return nullptr;
    }
    return t;
}

// A corpus table holds at most every n-gram of `n_refs` reference rows of `L` tokens (4 orders x min(L, 256) positions each), at a load of at most
// one half.  Growing frees the old slots after a device synchronisation; the slots' address is part of a step graph's key.
int cider_corpus_table_reserve(CiderTable* t, long n_refs, int L) {
    CAPB_REQUIRE(t != nullptr && t->corpus, "not a corpus CIDEr-D table");
    CAPB_REQUIRE(n_refs >= 0 && L >= 0, "bad reference shape");
    const long grams = (long)CIDER_N * n_refs * (L < CIDER_MAXL_LONG ? L : CIDER_MAXL_LONG);
    unsigned long long cap = 64;
    while (cap < (unsigned long long)(2 * grams + 2)) cap <<= 1;
    if (t->slots != nullptr && cap <= t->mask + 1) return 0;
    CAPB_CHECK_CUDA(cudaDeviceSynchronize());
    if (t->slots) CAPB_CHECK_CUDA(cudaFree(t->slots));
    t->slots = nullptr;
    t->mask = 0;
    CAPB_CHECK_CUDA(cudaMalloc(&t->slots, cap * sizeof(CiderSlot)));
    t->mask = cap - 1;
    return 0;
}

bool cider_table_is_corpus(const CiderTable* t) { return t != nullptr && t->corpus; }

void cider_table_key(const CiderTable* t, unsigned long long key[3]) {
    key[0] = t ? reinterpret_cast<unsigned long long>(t->slots) : 0ull;
    key[1] = t ? t->mask : 0ull;
    key[2] = t && t->corpus ? 1ull : 0ull;
}

namespace {

// ---- corpus document frequencies, built on the device in three launches: clear, insert, finalise

__global__ void corpus_clear_kernel(CiderSlot* __restrict__ slots, unsigned long long cap, unsigned int* used) {
    const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) *used = 0u;
    if (i >= cap) return;
    slots[i].key[0] = -2; slots[i].key[1] = -2; slots[i].key[2] = -2; slots[i].key[3] = -2;
    slots[i].idf = 0.0;
}

// the tokens of reference row r up to and including its first 0 (`with_eos`) or before it, at most min(L, 256)
__device__ __forceinline__ int ref_len(const int* __restrict__ refs, long r, int L, bool with_eos) {
    const int cols = L < CIDER_MAXL_LONG ? L : CIDER_MAXL_LONG;
    int len = 0;
    for (int j = 0; j < cols; ++j) {
        if (refs[r * L + j] == 0) return with_eos ? len + 1 : len;
        ++len;
    }
    return len;
}

// One CTA per image: every distinct n-gram of the image's references (set() over all of them, ciderD_scorer.py:143-147) adds `mult` -- the
// number of scored hypotheses (crefs entries) of the image -- to its document frequency.  References end as ref_len cuts them.  Thread items are (reference, order, position); an
// item inserts when no earlier item of the image holds the same n-gram.  A slot is claimed by swapping its key[0] from -2 (empty) to -3
// (being written); readers that meet -3 wait for the writer to publish key[0].  The occupied slots stay at most half the capacity (`used`),
// so every probe sequence, here and in the scoring kernels' lookups, reaches an empty slot.
__global__ void __launch_bounds__(256) corpus_insert_kernel(CiderSlot* __restrict__ slots, unsigned long long mask, unsigned int* used,
                                                            const int* __restrict__ refs, const int* __restrict__ ref_offsets, int L, double mult,
                                                            int with_eos) {
    const int img = blockIdx.x;
    const int r0 = ref_offsets[img], r1 = ref_offsets[img + 1];
    const int cols = L < CIDER_MAXL_LONG ? L : CIDER_MAXL_LONG;
    const long items = (long)(r1 - r0) * CIDER_N * cols;
    for (long it = threadIdx.x; it < items; it += blockDim.x) {
        const long r = r0 + it / (CIDER_N * cols);
        const int n = (int)((it / cols) % CIDER_N) + 1, p = (int)(it % cols);
        const int len = ref_len(refs, r, L, with_eos != 0);
        if (p + n > len) continue;
        const int* g = refs + r * L + p;
        bool first = true;
        for (long q = r0; q <= r && first; ++q) {
            const int lq = q == r ? p + n - 1 : ref_len(refs, q, L, with_eos != 0);          // earlier positions of this row, every position of earlier rows
            for (int j = 0; j + n <= lq && first; ++j) first = !same_gram(g, refs + q * L + j, n);
        }
        if (!first) continue;
        const int k0 = g[0], k1 = n > 1 ? g[1] : -1, k2 = n > 2 ? g[2] : -1, k3 = n > 3 ? g[3] : -1;
        unsigned long long h = cider_hash(k0, k1, k2, k3) & mask;
        for (unsigned long long probe = 0; probe <= mask; ++probe, h = (h + 1) & mask) {
            CiderSlot* s = slots + h;
            int cur = atomicCAS(&s->key[0], -2, -3);
            if (cur == -2) {
                if (atomicAdd(used, 1u) >= (unsigned int)((mask + 1) / 2)) { atomicExch(&s->key[0], -2); break; }    // over the reservation
                s->key[1] = k1; s->key[2] = k2; s->key[3] = k3;
                __threadfence();
                atomicExch(&s->key[0], k0);
                atomicAdd(&s->idf, mult);
                break;
            }
            while (cur == -3) cur = *(volatile int*)&s->key[0];
            __threadfence();
            const volatile int* vk = s->key;
            if (cur == k0 && vk[1] == k1 && vk[2] == k2 && vk[3] == k3) { atomicAdd(&s->idf, mult); break; }
        }
    }
}

// df -> log(ref_len) - log(max(1, df)), the weight the pickle table stores (cider_table_create)
__global__ void corpus_finalise_kernel(CiderSlot* __restrict__ slots, unsigned long long cap, double log_ref_len) {
    const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= cap || slots[i].key[0] == -2) return;
    const double df = slots[i].idf;
    slots[i].idf = log_ref_len - log(df > 1.0 ? df : 1.0);
}

// Builds the corpus table for one reward call over `hyps` scored hypotheses, `per_image` of them per image, and returns its log(ref_len) =
// log(hyps) (ciderD_scorer.py:182-186); a pickle table is left alone and returns its own.  The reward keeps each reference's closing 0
// (`with_eos`); coco-caption's Cider scores the words before it.
int corpus_build_launch(const CiderTable* t, int B, int hyps, int per_image, const int* refs, const int* ref_offsets, int L, double* log_ref_len,
                        cudaStream_t stream, bool with_eos = true) {
    if (!t->corpus) { *log_ref_len = t->log_ref_len; return 0; }
    CAPB_REQUIRE(t->slots != nullptr, "corpus CIDEr-D table without reserved slots (capb200_cider_table_reserve)");
    *log_ref_len = log((double)hyps);
    const unsigned long long cap = t->mask + 1;
    const unsigned int grid = (unsigned int)((cap + 255) / 256);
    corpus_clear_kernel<<<grid, 256, 0, stream>>>(t->slots, cap, t->used);
    CAPB_CHECK_CUDA(cudaGetLastError());
    corpus_insert_kernel<<<B, 256, 0, stream>>>(t->slots, t->mask, t->used, refs, ref_offsets, L, (double)per_image, with_eos ? 1 : 0);
    CAPB_CHECK_CUDA(cudaGetLastError());
    corpus_finalise_kernel<<<grid, 256, 0, stream>>>(t->slots, cap, *log_ref_len);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// Builds the tf-idf description of one caption held in shared memory.
//   gram index g = n * MAXL + p (order n+1 starting at position p);  w[g] = tf * idf for the first occurrence, else 0
//   nrm[n] = sqrt(sum w^2);  returns through `w`, `valid` (1 = distinct n-gram present)
// MAXL: CIDER_MAXL (captions and references of at most 64 tokens) or CIDER_MAXL_LONG (the long form, dispatched only past 64)
template <int MAXL>
__device__ void cider_vectorise(const CiderSlot* slots, unsigned long long mask, double log_ref_len, const int* tok, int len, double* w,
                                unsigned char* valid, double* nrm) {
    for (int g = threadIdx.x; g < CIDER_N * MAXL; g += blockDim.x) {
        const int n = g / MAXL + 1, p = g % MAXL;
        double wv = 0.0;
        unsigned char ok = 0;
        if (p + n <= len) {
            bool first = true;
            int tf = 0;
            for (int q = 0; q + n <= len; ++q) {
                if (same_gram(tok + p, tok + q, n)) {
                    if (q < p) { first = false; break; }
                    ++tf;
                }
            }
            if (first) {
                wv = (double)tf * cider_idf(slots, mask, log_ref_len, tok + p, n);
                ok = 1;
            }
        }
        w[g] = wv;
        valid[g] = ok;
    }
    __syncthreads();
    if (threadIdx.x < CIDER_N) {
        double s = 0.0;
        for (int p = 0; p < MAXL; ++p) {
            const int g = threadIdx.x * MAXL + p;
            if (valid[g]) s += w[g] * w[g];
        }
        nrm[threadIdx.x] = sqrt(s);
    }
    __syncthreads();
}

// one CTA per hypothesis: hyps 0..S-1 are the samples (image i / n), S..S+B-1 the greedy captions (image i - S).  Captions and references
// keep their closing 0 when `with_eos` (array_to_str, the reward form), else stop before it (the words coco-caption's Cider scores).
template <int MAXL>
__global__ void __launch_bounds__(256) cider_score_kernel(const CiderSlot* __restrict__ slots, unsigned long long mask, double log_ref_len,
                                                          const long long* __restrict__ sampled, int S, const long long* __restrict__ greedy, int B,
                                                          int T, const int* __restrict__ refs, const int* __restrict__ ref_offsets, int L,
                                                          double* __restrict__ scores, int with_eos) {
    __shared__ int h_tok[MAXL], r_tok[MAXL];
    __shared__ double h_w[CIDER_N * MAXL], r_w[CIDER_N * MAXL], contrib[CIDER_N * MAXL];
    __shared__ unsigned char h_valid[CIDER_N * MAXL], r_valid[CIDER_N * MAXL];
    __shared__ double h_nrm[CIDER_N], r_nrm[CIDER_N], acc[CIDER_N];
    __shared__ int h_len, r_len;
    const int hyp = blockIdx.x;
    const int n_per = (B > 0) ? S / B : 1;
    const int img = hyp < S ? hyp / n_per : hyp - S;
    const long long* src = hyp < S ? sampled + (long)hyp * T : greedy + (long)(hyp - S) * T;
    if (threadIdx.x == 0) {
        int len = 0;
        for (int i = 0; i < T && i < MAXL; ++i) {
            const int v = (int)src[i];
            if (v == 0 && !with_eos) break;
            h_tok[len++] = v;
            if (v == 0) break;
        }
        h_len = len;
    }
    __syncthreads();
    cider_vectorise<MAXL>(slots, mask, log_ref_len, h_tok, h_len, h_w, h_valid, h_nrm);
    const int hl = h_len > 1 ? h_len - 1 : 0;               // "length" = number of bigrams
    const int r0 = ref_offsets[img], r1 = ref_offsets[img + 1];
    double total = 0.0;                                       // only thread 0 uses it
    for (int r = r0; r < r1; ++r) {
        if (threadIdx.x == 0) {
            int len = 0;
            for (int i = 0; i < L && i < MAXL; ++i) {
                const int v = refs[(long)r * L + i];
                if (v == 0 && !with_eos) break;
                r_tok[len++] = v;
                if (v == 0) break;
            }
            r_len = len;
        }
        __syncthreads();
        cider_vectorise<MAXL>(slots, mask, log_ref_len, r_tok, r_len, r_w, r_valid, r_nrm);
        for (int g = threadIdx.x; g < CIDER_N * MAXL; g += blockDim.x) {
            double c = 0.0;
            if (h_valid[g]) {
                const int n = g / MAXL + 1, p = g % MAXL;
                double wr = 0.0;
                for (int q = 0; q + n <= r_len; ++q) {
                    const int gr = (n - 1) * MAXL + q;
                    if (r_valid[gr] && same_gram(h_tok + p, r_tok + q, n)) { wr = r_w[gr]; break; }
                }
                c = fmin(h_w[g], wr) * wr;
            }
            contrib[g] = c;
        }
        __syncthreads();
        if (threadIdx.x < CIDER_N) {
            const int n = threadIdx.x;
            double v = 0.0;
            for (int p = 0; p < MAXL; ++p) v += contrib[n * MAXL + p];
            if (h_nrm[n] != 0.0 && r_nrm[n] != 0.0) v /= (h_nrm[n] * r_nrm[n]);
            const int rl = r_len > 1 ? r_len - 1 : 0;
            const double delta = (double)(hl - rl);
            v *= exp(-(delta * delta) / (2.0 * 6.0 * 6.0));
            acc[n] = v;
        }
        __syncthreads();
        if (threadIdx.x == 0) total += (acc[0] + acc[1] + acc[2] + acc[3]) / (double)CIDER_N;
        __syncthreads();
    }
    if (threadIdx.x == 0) scores[hyp] = (r1 > r0) ? total / (double)(r1 - r0) * 10.0 : 0.0;
}

// BLEU-4 of one hypothesis, the per-sentence bleu_list[3] of BleuScorer.compute_score(option='closest') (bleu_scorer.py:26-80,184-260):
//   guess[k] = max(0, len_h - k);  correct[k] = sum over the hypothesis' distinct (k+1)-grams of min(count in h, max count in one reference)
//   bleu = (prod_k (correct[k] + 1e-15) / (guess[k] + 1e-9)) ** (1/4), times exp(1 - 1/ratio) when ratio = (len_h + 1e-15) / (reflen + 1e-9) < 1,
//   reflen = the reference length closest to len_h, the shorter one on a tie.  Lengths count words, the closing 0 included.
// One CTA per hypothesis, laid out as cider_score_kernel; thread g owns the n-gram of order g / MAXL + 1 starting at position g % MAXL (4 x 256 =
// 1024 threads in the long form: the CTA limit sets CAPB200_MAX_SEQ_LENGTH).  The image's
// references are staged in shared memory BLEU_REF_CHUNK at a time.  An image without references scores 0 (the Python layer refuses it).
// `with_eos` = 0 stops captions and references before their first 0 (the words coco-caption scores).  `scores` and `stats` may each be null;
// stats[hyp] gets correct 1..4-grams, the hypothesis length and the closest reference length (the layout of diversity.cu's BLEU statistics).
constexpr int BLEU_REF_CHUNK = 32;

template <int MAXL>
__global__ void __launch_bounds__(CIDER_N * MAXL) bleu_score_kernel(const long long* __restrict__ sampled, int S, const long long* __restrict__ greedy,
                                                                          int B, int T, const int* __restrict__ refs, const int* __restrict__ ref_offsets, int L,
                                                                          double* __restrict__ scores, int with_eos, int* __restrict__ stats) {
    __shared__ int h_tok[MAXL];
    __shared__ int r_tok[BLEU_REF_CHUNK][MAXL];
    __shared__ int r_len[BLEU_REF_CHUNK];
    __shared__ int correct[CIDER_N];
    __shared__ int h_len;
    const int hyp = blockIdx.x;
    const int n_per = (B > 0) ? S / B : 1;
    const int img = hyp < S ? hyp / n_per : hyp - S;
    const long long* src = hyp < S ? sampled + (long)hyp * T : greedy + (long)(hyp - S) * T;
    if (threadIdx.x == 0) {
        int len = 0;
        for (int i = 0; i < T && i < MAXL; ++i) {
            const int v = (int)src[i];
            if (v == 0 && !with_eos) break;
            h_tok[len++] = v;
            if (v == 0) break;
        }
        h_len = len;
    }
    if (threadIdx.x < CIDER_N) correct[threadIdx.x] = 0;
    __syncthreads();
    const int hl = h_len;
    const int n = threadIdx.x / MAXL + 1, p = threadIdx.x % MAXL;
    // counted by its first occurrence only: tf = how often the n-gram occurs in the hypothesis
    bool first = p + n <= hl;
    int tf = 0;
    for (int q = 0; first && q + n <= hl; ++q) {
        if (same_gram(h_tok + p, h_tok + q, n)) {
            if (q < p) first = false;
            else ++tf;
        }
    }
    int max_ref = 0;                                    // the n-gram's largest count in a single reference
    int best_len = -1, best_diff = 0;                   // closest reference length (thread 0)
    const int r0 = ref_offsets[img], r1 = ref_offsets[img + 1];
    const int cols = L < MAXL ? L : MAXL;
    for (int c0 = r0; c0 < r1; c0 += BLEU_REF_CHUNK) {
        const int cnt = r1 - c0 < BLEU_REF_CHUNK ? r1 - c0 : BLEU_REF_CHUNK;
        __syncthreads();                                // the previous chunk has been read
        for (int i = threadIdx.x; i < cnt * MAXL; i += blockDim.x) {
            const int r = i / MAXL, j = i % MAXL;
            r_tok[r][j] = j < cols ? refs[(long)(c0 + r) * L + j] : 0;
        }
        __syncthreads();
        if (threadIdx.x < cnt) {
            int len = 0;
            for (int j = 0; j < cols; ++j) {
                if (r_tok[threadIdx.x][j] == 0) { len += with_eos ? 1 : 0; break; }
                ++len;
            }
            r_len[threadIdx.x] = len;
        }
        __syncthreads();
        if (first) {
            for (int r = 0; r < cnt; ++r) {
                int c = 0;
                for (int q = 0; q + n <= r_len[r]; ++q) c += same_gram(h_tok + p, r_tok[r] + q, n) ? 1 : 0;
                max_ref = c > max_ref ? c : max_ref;
            }
        }
        if (threadIdx.x == 0) {
            for (int r = 0; r < cnt; ++r) {
                const int d = abs(r_len[r] - hl);
                if (best_len < 0 || d < best_diff || (d == best_diff && r_len[r] < best_len)) { best_len = r_len[r]; best_diff = d; }
            }
        }
    }
    if (first) atomicAdd(&correct[n - 1], tf < max_ref ? tf : max_ref);
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        if (best_len >= 0) {
            double prod = 1.0;
            for (int k = 0; k < CIDER_N; ++k) {
                const int guess = hl - k > 0 ? hl - k : 0;
                prod *= ((double)correct[k] + 1e-15) / ((double)guess + 1e-9);
            }
            s = pow(prod, 0.25);
            const double ratio = ((double)hl + 1e-15) / ((double)best_len + 1e-9);
            if (ratio < 1.0) s *= exp(1.0 - 1.0 / ratio);
        }
        if (scores) scores[hyp] = s;
        if (stats) {
            int* st = stats + (long)hyp * 6;
            for (int k = 0; k < CIDER_N; ++k) st[k] = correct[k];
            st[4] = hl;
            st[5] = best_len;
        }
    }
}

// score = cider_weight * CIDEr-D + bleu_weight * BLEU-4 in place over `scores` (which holds CIDEr-D when its weight is > 0), in float64 as
// rewards.py:74,112 computes it; a term whose weight is <= 0 was not computed and contributes weight * 0.  Rounded operations keep the
// compiler from contracting the sum into an FMA that numpy does not perform.
__global__ void reward_combine_kernel(double* __restrict__ scores, const double* __restrict__ bleu, int hyps, double wc, double wb) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= hyps) return;
    const double c = __dmul_rn(wc, wc > 0.0 ? scores[i] : 0.0);
    const double b = __dmul_rn(wb, wb > 0.0 ? bleu[i] : 0.0);
    scores[i] = __dadd_rn(c, b);
}

__global__ void cider_reward_kernel(const double* __restrict__ scores, int S, int B, float* __restrict__ reward, long ld, int cols) {
    const int i = blockIdx.x;
    const int n_per = S / B;
    const float rwd = (float)(scores[i] - scores[S + i / n_per]);     // fp64 difference, then the .to(float32) of loss_wrapper.py:71
    for (int c = threadIdx.x; c < cols; c += blockDim.x) reward[(long)i * ld + c] = rwd;
}

// new_self_critical (losses.py:168-187): reward_i = s_i - mean of the image's other samples, in fp32 after scores.type_as(input) (:62)
__global__ void cider_reward_loo_kernel(const double* __restrict__ scores, int n_per, float* __restrict__ reward, long ld, int cols) {
    const int i = blockIdx.x;
    const int first = (i / n_per) * n_per;
    float sum = 0.f;
    for (int j = 0; j < n_per; ++j) sum += (float)scores[first + j];
    const float s = (float)scores[i];
    const float rwd = s - (sum - s) / (float)(n_per - 1);
    for (int c = threadIdx.x; c < cols; c += blockDim.x) reward[(long)i * ld + c] = rwd;
}

// RewardCriterion (losses.py:22-37): single CTA, deterministic tree reduction
__global__ void __launch_bounds__(256) reward_criterion_fwd_kernel(const float* __restrict__ lp, long ld_row, long ld_t, const long long* __restrict__ seq,
                                                                   const float* __restrict__ reward, int N, int T, float* loss_mean,
                                                                   float* loss_rows, float* mask_sum) {
    __shared__ float s_out[256], s_msk[256];
    float o_acc = 0.f, m_acc = 0.f;
    for (int n = threadIdx.x; n < N; n += blockDim.x) {
        float ro = 0.f, rm = 0.f;
        for (int t = 0; t < T; ++t) {
            const float m = (t == 0 || seq[(long)n * T + t - 1] > 0) ? 1.f : 0.f;
            const long long tok = seq[(long)n * T + t];
            const float v = -lp[(long)n * ld_row + (long)t * ld_t + tok] * reward[(long)n * T + t] * m;
            ro += v;
            rm += m;
        }
        if (loss_rows) loss_rows[n] = ro / rm;
        o_acc += ro;
        m_acc += rm;
    }
    s_out[threadIdx.x] = o_acc;
    s_msk[threadIdx.x] = m_acc;
    __syncthreads();
    for (int w = 128; w > 0; w >>= 1) {
        if (threadIdx.x < w) { s_out[threadIdx.x] += s_out[threadIdx.x + w]; s_msk[threadIdx.x] += s_msk[threadIdx.x + w]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        if (loss_mean) *loss_mean = s_out[0] / s_msk[0];
        if (mask_sum) *mask_sum = s_msk[0];
    }
}

__global__ void reward_criterion_bwd_kernel(const long long* __restrict__ seq, const float* __restrict__ reward, int N, int T,
                                            const float* __restrict__ mask_sum, float upstream, float* __restrict__ grad, long ld_row, long ld_t) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N * T) return;
    const int n = i / T, t = i % T;
    const float m = (t == 0 || seq[(long)n * T + t - 1] > 0) ? 1.f : 0.f;
    const long long tok = seq[i];
    grad[(long)n * ld_row + (long)t * ld_t + tok] = -reward[i] * m / (*mask_sum) * upstream;
}

// The reward from the hypothesis scores: the greedy difference (greedy != nullptr) or the leave-one-out baseline.
int baseline_reward_launch(const double* scores, int S, const long long* greedy, int B, float* reward, long ld_reward, int reward_cols, cudaStream_t stream) {
    if (reward == nullptr || S == 0) return 0;
    if (greedy != nullptr) {
        cider_reward_kernel<<<S, 32, 0, stream>>>(scores, S, B, reward, ld_reward, reward_cols);
    } else {
        CAPB_REQUIRE(S / B >= 2, "the leave-one-out baseline needs at least two samples per image");
        cider_reward_loo_kernel<<<S, 32, 0, stream>>>(scores, S / B, reward, ld_reward, reward_cols);
    }
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int check_reward_shapes(int S, int B, int T, int L) {
    CAPB_REQUIRE(B > 0 && S % B == 0, "sample rows must be a multiple of the image count");
    CAPB_REQUIRE(T <= CIDER_MAXL_LONG && L <= CIDER_MAXL_LONG, "caption or reference length above 256 tokens (CAPB200_MAX_SEQ_LENGTH)");
    return 0;
}

// the short kernels up to 64 tokens (hypotheses and references), the long ones past it
bool long_form(int T, int L) { return T > CIDER_MAXL || L > CIDER_MAXL; }

void cider_score_launch(const CiderTable* t, double log_ref_len, const long long* sampled, int S, const long long* greedy, int B, int T, const int* refs,
                        const int* ref_offsets, int L, double* scores, int hyps, cudaStream_t stream, bool with_eos = true) {
    const int eos = with_eos ? 1 : 0;
    if (long_form(T, L))
        cider_score_kernel<CIDER_MAXL_LONG><<<hyps, 256, 0, stream>>>(t->slots, t->mask, log_ref_len, sampled, S, greedy, B, T, refs, ref_offsets, L, scores, eos);
    else
        cider_score_kernel<CIDER_MAXL><<<hyps, 256, 0, stream>>>(t->slots, t->mask, log_ref_len, sampled, S, greedy, B, T, refs, ref_offsets, L, scores, eos);
}

void bleu_score_launch(const long long* sampled, int S, const long long* greedy, int B, int T, const int* refs, const int* ref_offsets, int L, double* scores,
                       int hyps, cudaStream_t stream, bool with_eos = true, int* stats = nullptr) {
    const int eos = with_eos ? 1 : 0;
    if (long_form(T, L))
        bleu_score_kernel<CIDER_MAXL_LONG><<<hyps, CIDER_N * CIDER_MAXL_LONG, 0, stream>>>(sampled, S, greedy, B, T, refs, ref_offsets, L, scores, eos, stats);
    else
        bleu_score_kernel<CIDER_MAXL><<<hyps, CIDER_N * CIDER_MAXL, 0, stream>>>(sampled, S, greedy, B, T, refs, ref_offsets, L, scores, eos, stats);
}

}  // namespace

int cider_reward_launch(const CiderTable* t, const long long* sampled, int S, const long long* greedy, int B, int T, const int* refs,
                        const int* ref_offsets, int L, double* scores, float* reward, long ld_reward, int reward_cols, cudaStream_t stream) {
    CAPB_REQUIRE(t != nullptr, "CIDEr-D table not initialised (init_scorer)");
    if (check_reward_shapes(S, B, T, L)) return 1;
    // greedy == nullptr: score the samples only; the reward baseline is then the mean of the image's other samples
    const int hyps = greedy != nullptr ? S + B : S;
    if (hyps == 0) return 0;
    double log_ref_len = 0.0;
    if (corpus_build_launch(t, B, hyps, hyps / B, refs, ref_offsets, L, &log_ref_len, stream)) return 1;
    cider_score_launch(t, log_ref_len, sampled, S, greedy, B, T, refs, ref_offsets, L, scores, hyps, stream);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return baseline_reward_launch(scores, S, greedy, B, reward, ld_reward, reward_cols, stream);
}

int bleu_scores_launch(const long long* sampled, int S, const long long* greedy, int B, int T, const int* refs, const int* ref_offsets, int L,
                       double* scores, cudaStream_t stream) {
    if (check_reward_shapes(S, B, T, L)) return 1;
    const int hyps = greedy != nullptr ? S + B : S;
    if (hyps == 0) return 0;
    bleu_score_launch(sampled, S, greedy, B, T, refs, ref_offsets, L, scores, hyps, stream);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// coco-caption's Cider() and the Bleu(4) statistics over the words of seqs[S, T] (the ids before the first 0), per_image = S / n_images
// consecutive captions per image, against references cut the same way.  Cider's document frequencies count each image once whatever
// per_image is, with ref_len = log(n_images) (cider_scorer.py:96-107,165: one Cider call scores one caption per image).  `t` is a corpus
// table reserved for the references.
int coco_cider_bleu_launch(const CiderTable* t, const long long* seqs, int S, int n_images, int T, const int* refs, const int* ref_offsets, int L,
                           double* cider, int* bleu_stats, cudaStream_t stream) {
    CAPB_REQUIRE(t != nullptr && t->corpus, "the caption metrics build their document frequencies in a corpus CIDEr table");
    if (check_reward_shapes(S, n_images, T, L)) return 1;
    double log_ref_len = 0.0;
    if (corpus_build_launch(t, n_images, n_images, 1, refs, ref_offsets, L, &log_ref_len, stream, false)) return 1;
    cider_score_launch(t, log_ref_len, seqs, S, nullptr, n_images, T, refs, ref_offsets, L, cider, S, stream, false);
    CAPB_CHECK_CUDA(cudaGetLastError());
    bleu_score_launch(seqs, S, nullptr, n_images, T, refs, ref_offsets, L, nullptr, S, stream, false, bleu_stats);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int weighted_reward_launches(double w_cider, double w_bleu, bool with_reward) {
    return (w_cider > 0.0) + (w_bleu > 0.0) + 1 + (with_reward ? 1 : 0);
}

int corpus_build_launches(const CiderTable* t) { return t != nullptr && t->corpus ? 3 : 0; }

int weighted_reward_launch(const CiderTable* t, double w_cider, double w_bleu, const long long* sampled, int S, const long long* greedy, int B, int T,
                           const int* refs, const int* ref_offsets, int L, double* scores, double* bleu, float* reward, long ld_reward, int reward_cols,
                           cudaStream_t stream) {
    CAPB_REQUIRE(std::isfinite(w_cider) && std::isfinite(w_bleu), "reward weights must be finite");
    CAPB_REQUIRE(w_cider <= 0.0 || t != nullptr, "CIDEr-D table not initialised (init_scorer)");
    CAPB_REQUIRE(w_bleu <= 0.0 || bleu != nullptr, "the BLEU-4 term needs its score buffer");
    if (check_reward_shapes(S, B, T, L)) return 1;
    const int hyps = greedy != nullptr ? S + B : S;
    if (hyps == 0) return 0;
    if (w_cider > 0.0) {
        double log_ref_len = 0.0;
        if (corpus_build_launch(t, B, hyps, hyps / B, refs, ref_offsets, L, &log_ref_len, stream)) return 1;
        cider_score_launch(t, log_ref_len, sampled, S, greedy, B, T, refs, ref_offsets, L, scores, hyps, stream);
        CAPB_CHECK_CUDA(cudaGetLastError());
    }
    if (w_bleu > 0.0 && bleu_scores_launch(sampled, S, greedy, B, T, refs, ref_offsets, L, bleu, stream)) return 1;
    reward_combine_kernel<<<cdiv(hyps, 256), 256, 0, stream>>>(scores, bleu, hyps, w_cider, w_bleu);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return baseline_reward_launch(scores, S, greedy, B, reward, ld_reward, reward_cols, stream);
}

int reward_criterion_fwd_launch(const float* logprobs, long ld_row, long ld_t, const long long* seq, const float* reward, int N, int T,
                                float* loss_mean, float* loss_rows, float* mask_sum, cudaStream_t stream) {
    reward_criterion_fwd_kernel<<<1, 256, 0, stream>>>(logprobs, ld_row, ld_t, seq, reward, N, T, loss_mean, loss_rows, mask_sum);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int reward_criterion_bwd_launch(const long long* seq, const float* reward, int N, int T, const float* mask_sum, float upstream,
                                float* grad, long ld_row, long ld_t, cudaStream_t stream) {
    if (N * T <= 0) return 0;
    reward_criterion_bwd_kernel<<<cdiv(N * T, 256), 256, 0, stream>>>(seq, reward, N, T, mask_sum, upstream, grad, ld_row, ld_t);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace capb200
