// Language evaluation on the device: coco-caption's Bleu(4), Rouge() and Cider() over token ids.
//
// Replaces the pure-Python scorers COCOEvalCap runs after the PTB tokenizer (coco-caption/pycocoevalcap):
//   Bleu(4)    bleu/bleu_scorer.py:26-86,201-266   option 'closest': per-sentence bleu_list and the corpus score
//   Rouge()    rouge/rouge.py:15-77                LCS precision / recall maxima over the references, F with beta = 1.2
//   Cider()    cider/cider_scorer.py:96-184        clipped tf-idf cosine with the sigma = 6 length penalty, x 10
// A caption is the string of its ids before the first 0, joined by single spaces; references are the image's 0-padded label rows cut the
// same way.  Bleu and Cider split on whitespace, so an empty caption has no words; Rouge splits on " ", so it has one empty word, which
// only an empty reference matches.  Every score is float64.
#include <cmath>
#include <vector>

#include "cider_table.cuh"
#include "common.cuh"
#include "engine_common.cuh"

namespace capb200 {

namespace {

constexpr int ROUGE_THREADS = 32;     // one warp per caption, one lane per reference
constexpr int COCO_BLEU_STATS = 6;    // per caption: correct 1..4-grams, length, closest reference length (reward.cu's bleu_score_kernel)
constexpr int EMPTY_WORD = -1;        // the '' token of "".split(" ")

// ---- ROUGE-L: one warp per caption
//
// Lane l takes references l, l + 32, ...: the LCS of the caption and the reference (my_lcs; it is symmetric) by the row-by-row dynamic
// programme over the caption's positions, held in the lane's own row of shared memory [T + 1].  prec = lcs / caption words and
// rec = lcs / reference words are maximised separately over the references; score = (1 + b^2) p r / (r + b^2 p), 0 when either is 0.
// Rounded operations keep the compiler from contracting the score into an FMA that Python does not perform.
__global__ void __launch_bounds__(ROUGE_THREADS) rouge_kernel(const long long* __restrict__ seqs, int per_image, int T, const int* __restrict__ refs,
                                                             const int* __restrict__ ref_offsets, int L, double* __restrict__ out) {
    extern __shared__ int rouge_smem[];
    int* cap = rouge_smem;                                              // [T]
    int* row = cap + T + threadIdx.x * (T + 1);                         // [32][T + 1]
    const int s = blockIdx.x, img = s / per_image, lane = threadIdx.x;
    int m = 0;                                                          // caption words; every lane reads the same row
    for (int j = 0; j < T; ++j) {
        const int v = (int)seqs[(long)s * T + j];
        if (v == 0) break;
        if (lane == 0) cap[m] = v;
        ++m;
    }
    if (m == 0) {
        if (lane == 0) cap[0] = EMPTY_WORD;
        m = 1;
    }
    __syncwarp();
    const int r0 = ref_offsets[img], r1 = ref_offsets[img + 1];
    const int rcols = L < CIDER_MAXL_LONG ? L : CIDER_MAXL_LONG;
    double prec = 0.0, rec = 0.0;
    for (int r = r0 + lane; r < r1; r += ROUGE_THREADS) {
        for (int j = 0; j <= m; ++j) row[j] = 0;
        int n = 0;
        for (int i = 0; i <= rcols; ++i) {
            int x = i < rcols ? refs[(long)r * L + i] : 0;
            if (x == 0) {
                if (n > 0) break;
                x = EMPTY_WORD;                                         // an empty reference: one '' word
            }
            ++n;
            int diag = 0;
            for (int j = 1; j <= m; ++j) {
                const int up = row[j];
                row[j] = x == cap[j - 1] ? diag + 1 : max(up, row[j - 1]);
                diag = up;
            }
            if (x == EMPTY_WORD) break;
        }
        const int lcs = row[m];
        prec = fmax(prec, (double)lcs / (double)m);
        rec = fmax(rec, (double)lcs / (double)n);
    }
    for (int o = 16; o > 0; o >>= 1) {
        prec = fmax(prec, __shfl_xor_sync(0xffffffffu, prec, o));
        rec = fmax(rec, __shfl_xor_sync(0xffffffffu, rec, o));
    }
    if (lane == 0) {
        const double b2 = __dmul_rn(1.2, 1.2);
        double score = 0.0;
        if (prec != 0.0 && rec != 0.0)
            score = __dmul_rn(__dmul_rn(__dadd_rn(1.0, b2), prec), rec) / __dadd_rn(rec, __dmul_rn(b2, prec));
        out[s] = score;
    }
}

// Per-sentence BLEU-1..4 (bleu_list of BleuScorer.compute_score) from the statistics: the running product of (correct + 1e-15) /
// (guess + 1e-9), its (k+1)-th root, times exp(1 - 1/ratio) when ratio = (length + 1e-15) / (closest reference length + 1e-9) < 1.
__global__ void sentence_bleu_kernel(const int* __restrict__ stats, int S, double* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= S) return;
    const int* st = stats + (long)i * COCO_BLEU_STATS;
    const int hl = st[4];
    const double ratio = ((double)hl + 1e-15) / ((double)st[5] + 1e-9);
    double b = 1.0;
    for (int k = 0; k < CIDER_N; ++k) {
        const int guess = hl - k > 0 ? hl - k : 0;
        b *= ((double)st[k] + 1e-15) / ((double)guess + 1e-9);
        double v = pow(b, 1.0 / (k + 1));
        if (ratio < 1.0) v *= exp(1.0 - 1.0 / ratio);
        out[(long)i * CIDER_N + k] = v;
    }
}

int check_coco_shapes(int n_images, int per_image, int T, int L) {
    CAPB_REQUIRE(n_images >= 1, "no images to score");
    CAPB_REQUIRE(per_image >= 1, "at least one caption per image");
    CAPB_REQUIRE((long)n_images * per_image <= 0x7fffffffL, "too many captions");
    CAPB_REQUIRE(T >= 1 && T <= CAPB200_MAX_SEQ_LENGTH, "caption length between 1 and 256 tokens (CAPB200_MAX_SEQ_LENGTH)");
    CAPB_REQUIRE(L >= 1 && L <= CAPB200_MAX_SEQ_LENGTH, "reference length between 1 and 256 tokens (CAPB200_MAX_SEQ_LENGTH)");
    return 0;
}

}  // namespace

int coco_scores_launch(CiderTable* t, const long long* seqs, int n_images, int per_image, int T, const int* refs, const int* ref_offsets, int L,
                       double* out_bleu, double* out_corpus_bleu, double* out_rouge, double* out_cider, int* ws_stats, cudaStream_t stream) {
    CAPB_REQUIRE(t != nullptr && t->corpus, "the caption metrics need a corpus CIDEr table (capb200_cider_corpus_table_create)");
    if (check_coco_shapes(n_images, per_image, T, L)) return 1;
    // every image needs a reference (the scorers assert it): the offsets are read back and checked before any launch
    static thread_local std::vector<int> offs;
    offs.resize((size_t)n_images + 1);
    CAPB_CHECK_CUDA(cudaMemcpyAsync(offs.data(), ref_offsets, offs.size() * sizeof(int), cudaMemcpyDeviceToHost, stream));
    CAPB_CHECK_CUDA(cudaStreamSynchronize(stream));
    CAPB_REQUIRE(offs[0] == 0, "reference offsets must start at 0");
    for (int i = 0; i < n_images; ++i) CAPB_REQUIRE(offs[i + 1] > offs[i], "every image needs at least one reference");
    if (cider_corpus_table_reserve(t, offs[n_images], L)) return 1;
    const int S = n_images * per_image;
    if (coco_cider_bleu_launch(t, seqs, S, n_images, T, refs, ref_offsets, L, out_cider, ws_stats, stream)) return 1;
    sentence_bleu_kernel<<<cdiv(S, 256), 256, 0, stream>>>(ws_stats, S, out_bleu);
    CAPB_CHECK_CUDA(cudaGetLastError());
    if (corpus_bleu_launch(ws_stats, n_images, per_image, out_corpus_bleu, stream)) return 1;
    const size_t smem = ((size_t)T + (size_t)ROUGE_THREADS * (T + 1)) * sizeof(int);
    CAPB_CHECK_CUDA(cudaFuncSetAttribute(rouge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    rouge_kernel<<<S, ROUGE_THREADS, smem, stream>>>(seqs, per_image, T, refs, ref_offsets, L, out_rouge);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace capb200

using namespace capb200;

extern "C" {

int capb200_coco_scores(capb200_cider_table* t, const long long* seqs, int n_images, int per_image, int T, const int* refs, const int* ref_offsets,
                        int L, double* out_bleu, double* out_corpus_bleu, double* out_rouge, double* out_cider, int* ws_stats, void* stream) {
    CAPB_REQUIRE(t != nullptr && seqs && refs && ref_offsets && out_bleu && out_corpus_bleu && out_rouge && out_cider && ws_stats, "null argument");
    return coco_scores_launch(t->t, seqs, n_images, per_image, T, refs, ref_offsets, L, out_bleu, out_corpus_bleu, out_rouge, out_cider, ws_stats,
                              static_cast<cudaStream_t>(stream));
}

}  // extern "C"
