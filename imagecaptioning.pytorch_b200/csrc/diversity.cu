// Diversity of caption sets on the device: self-CIDEr matrices and their eigenvalue score, Div-n, gDiv-1 and mutual BLEU.
//
// Replaces the host Python the reference runs to score the n captions it generates per image:
//   get_self_cider_scores      captioning/utils/rewards.py:116-138   (Cider(df=cached_tokens).my_self_cider + numpy eigvalsh per image)
//   eval_self_cider            captioning/utils/eval_multi.py:177-217
//   my_get_self_cider          cider/pyciderevalcap/cider/cider_scorer.py:240-258, counts2vec / sim of the same file (plain CIDEr, not CIDEr-D)
//   eval_div_stats             captioning/utils/eval_multi.py:121-175, compute_div_n / compute_global_div_n of captioning/utils/div_utils.py
// Captions are rows of token ids, n consecutive rows per image.  A self-CIDEr caption is cut through its first 0 (array_to_str, the reward
// form) or before it (the decoded words of eval_self_cider); Div-n and mutual BLEU always work on the words, before the first 0.
// Every sum is float64 and each CTA reduces in a fixed order, so two calls give the same bits.
#include <cmath>

#include "cider_table.cuh"
#include "common.cuh"
#include "engine_common.cuh"

namespace capb200 {

constexpr int DIV_MAXN = 32;          // captions per image: one warp's Jacobi sweep, one lane per row
constexpr int DIV_THREADS = 256;
constexpr int DIV_BLEU_STATS = 6;     // per caption: correct 1..4-grams, length, closest reference length

namespace {

// the tokens of row r: through the first 0 when `with_eos`, else before it; at most min(T, 64)
__device__ __forceinline__ int load_caption(const long long* __restrict__ seqs, long r, int T, bool with_eos, int* dst) {
    const int cols = T < CIDER_MAXL ? T : CIDER_MAXL;
    int len = 0;
    for (int j = 0; j < cols; ++j) {
        const int v = (int)seqs[r * T + j];
        if (v == 0 && !with_eos) break;
        dst[len++] = v;
        if (v == 0) break;
    }
    return len;
}

// ---- self-CIDEr matrix: one CTA per image
//
// For caption c, order k and position p, w[c][k][p] is counts2vec's tf * idf at the n-gram's first position in the caption (0 elsewhere) and
// gid[c][k][p] names the n-gram image-wide: the flat index c' * 64 + p' of its first occurrence over the image's captions, -1 when p is not
// the first position in caption c.  sim (cider_scorer.py:51-77) of captions i and j at order k sums w_i * w_j over i's distinct n-grams in
// the order counts2vec met them (positions ascending), then divides by both norms when neither is 0; the entry is 10 * their mean over k.
// There is no clipping and no length penalty: this is CIDEr, not CIDEr-D.  Rounded operations keep the compiler from contracting a product
// and a sum into an FMA that numpy does not perform.
__global__ void __launch_bounds__(DIV_THREADS) self_cider_matrix_kernel(const CiderSlot* __restrict__ slots, unsigned long long mask, double log_ref_len,
                                                                        const long long* __restrict__ seqs, int n, int T, int with_eos,
                                                                        double* __restrict__ out_mat) {
    extern __shared__ double smem[];
    double* w = smem;                                               // [n][4][64]
    double* nrm = w + (size_t)n * CIDER_N * CIDER_MAXL;             // [n][4]
    int* gid = reinterpret_cast<int*>(nrm + n * CIDER_N);          // [n][4][64]
    int* tok = gid + n * CIDER_N * CIDER_MAXL;                      // [n][64]
    int* len = tok + n * CIDER_MAXL;                                // [n]
    const int img = blockIdx.x;
    if (threadIdx.x < n) len[threadIdx.x] = load_caption(seqs, (long)img * n + threadIdx.x, T, with_eos != 0, tok + threadIdx.x * CIDER_MAXL);
    __syncthreads();
    for (int it = threadIdx.x; it < n * CIDER_N * CIDER_MAXL; it += blockDim.x) {
        const int c = it / (CIDER_N * CIDER_MAXL), k = (it / CIDER_MAXL) % CIDER_N, p = it % CIDER_MAXL, g = k + 1;
        const int* t = tok + c * CIDER_MAXL;
        double wv = 0.0;
        int id = -1;
        if (p + g <= len[c]) {
            bool first = true;
            int tf = 0;
            for (int q = 0; q + g <= len[c]; ++q) {
                if (same_gram(t + p, t + q, g)) {
                    if (q < p) { first = false; break; }
                    ++tf;
                }
            }
            if (first) {
                wv = __dmul_rn((double)tf, cider_idf(slots, mask, log_ref_len, t + p, g));
                id = c * CIDER_MAXL + p;
                for (int c2 = 0; c2 < c && id == c * CIDER_MAXL + p; ++c2)
                    for (int q = 0; q + g <= len[c2]; ++q)
                        if (same_gram(t + p, tok + c2 * CIDER_MAXL + q, g)) { id = c2 * CIDER_MAXL + q; break; }
            }
        }
        w[it] = wv;
        gid[it] = id;
    }
    __syncthreads();
    if (threadIdx.x < n * CIDER_N) {
        const double* wr = w + threadIdx.x * CIDER_MAXL;
        double s = 0.0;
        for (int p = 0; p < CIDER_MAXL; ++p) s = __dadd_rn(s, __dmul_rn(wr[p], wr[p]));
        nrm[threadIdx.x] = sqrt(s);
    }
    __syncthreads();
    for (int pr = threadIdx.x; pr < n * n; pr += blockDim.x) {
        const int i = pr / n, j = pr % n;
        double total = 0.0;
        for (int k = 0; k < CIDER_N; ++k) {
            const int* gi = gid + (i * CIDER_N + k) * CIDER_MAXL;
            const int* gj = gid + (j * CIDER_N + k) * CIDER_MAXL;
            const double* wi = w + (i * CIDER_N + k) * CIDER_MAXL;
            const double* wj = w + (j * CIDER_N + k) * CIDER_MAXL;
            const int li = len[i] - k, lj = len[j] - k;
            double v = 0.0;
            for (int p = 0; p < li; ++p) {
                if (gi[p] < 0) continue;
                double wr = 0.0;
                for (int q = 0; q < lj; ++q) if (gj[q] == gi[p]) { wr = wj[q]; break; }
                v = __dadd_rn(v, __dmul_rn(wi[p], wr));
            }
            const double ni = nrm[i * CIDER_N + k], nj = nrm[j * CIDER_N + k];
            if (ni != 0.0 && nj != 0.0) v /= __dmul_rn(ni, nj);
            total = __dadd_rn(total, v);
        }
        out_mat[((long)img * n + i) * n + j] = __dmul_rn(total / (double)CIDER_N, 10.0);
    }
}

// ---- eigenvalue diversity: one warp per image
//
// get_div(eigvalsh(M / 10)) (rewards.py:130-133): -log(sqrt(l_max) / sum sqrt(l)) / log(n) over the eigenvalues clipped at 0.  eigvalsh reads
// the lower triangle only, so the warp does too: A[r][c] = A[c][r] = M[max(r, c)][min(r, c)] / 10.  Cyclic Jacobi in float64: sweeps over the
// pairs (p, q) in row order, each rotation zeroing A[p][q] (the rotation of Numerical Recipes' jacobi, lane r updating row / column r), until
// a sweep starts with every off-diagonal entry at most 1e-18 times the largest diagonal magnitude, or after 64 sweeps.  The eigenvalues are
// summed in ascending order, as numpy returns them.
__global__ void __launch_bounds__(32) self_cider_div_kernel(const double* __restrict__ mat, int n, double* __restrict__ out_score) {
    __shared__ double a[DIV_MAXN][DIV_MAXN + 1];
    const int img = blockIdx.x, lane = threadIdx.x;
    const double* m = mat + (long)img * n * n;
    if (lane < n)
        for (int c = 0; c < n; ++c) a[lane][c] = (lane >= c ? m[lane * n + c] : m[c * n + lane]) / 10.0;
    __syncwarp();
    for (int sweep = 0; sweep < 64; ++sweep) {
        double off = 0.0, diag = 0.0;
        for (int r = 0; r < n; ++r) {
            diag = fmax(diag, fabs(a[r][r]));
            for (int c = r + 1; c < n; ++c) off = fmax(off, fabs(a[r][c]));
        }
        if (off <= 1e-18 * diag || off == 0.0) break;
        for (int p = 0; p < n - 1; ++p) {
            for (int q = p + 1; q < n; ++q) {
                const double apq = a[p][q];
                if (apq == 0.0) continue;
                const double theta = (a[q][q] - a[p][p]) / (2.0 * apq);
                const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                const double c = 1.0 / sqrt(t * t + 1.0), s = t * c, tau = s / (1.0 + c);
                const double app = a[p][p], aqq = a[q][q];
                double gr = 0.0, hr = 0.0;
                if (lane < n && lane != p && lane != q) { gr = a[lane][p]; hr = a[lane][q]; }
                __syncwarp();
                if (lane < n && lane != p && lane != q) {
                    const double np = gr - s * (hr + gr * tau), nq = hr + s * (gr - hr * tau);
                    a[lane][p] = np; a[p][lane] = np;
                    a[lane][q] = nq; a[q][lane] = nq;
                }
                if (lane == 0) {
                    a[p][p] = app - t * apq;
                    a[q][q] = aqq + t * apq;
                    a[p][q] = 0.0; a[q][p] = 0.0;
                }
                __syncwarp();
            }
        }
    }
    if (lane == 0) {
        double ev[DIV_MAXN];
        for (int r = 0; r < n; ++r) {
            const double v = a[r][r] > 0.0 ? a[r][r] : 0.0;          // np.clip(eigvals, 0, None)
            int at = r;
            while (at > 0 && ev[at - 1] > v) { ev[at] = ev[at - 1]; --at; }
            ev[at] = v;
        }
        double sum = 0.0;
        for (int r = 0; r < n; ++r) sum += sqrt(ev[r]);
        out_score[img] = -log(sqrt(ev[n - 1]) / sum) / log((double)n);
    }
}

// ---- Div-1, Div-2 and the per-caption mutual BLEU statistics: one CTA per image
//
// compute_div_n (div_utils.py:10-21): distinct n-grams of the image's captions (n-grams inside one caption) / (1e-6 + total words).
// Mutual BLEU (eval_multi.py:140-152) scores caption j against the image's other n - 1 captions with Bleu(4) (bleu_scorer.py, closest
// reference length): correct[k] = sum over j's distinct (k+1)-grams of min(count in j, max count in one other caption), the shorter length on
// a tie.  The per-sentence BLEU-2 (scores[1]) is written here; the statistics go out for the corpus BLEU of each leave-one-out round.
__global__ void __launch_bounds__(DIV_THREADS) div_stats_kernel(const long long* __restrict__ seqs, int n, int T, double* __restrict__ out_div1,
                                                                double* __restrict__ out_div2, double* __restrict__ out_bleu2, int* __restrict__ stats) {
    __shared__ int tok[DIV_MAXN][CIDER_MAXL];
    __shared__ int len[DIV_MAXN];
    __shared__ int correct[DIV_MAXN][CIDER_N];
    __shared__ int distinct[2], words;
    const int img = blockIdx.x;
    if (threadIdx.x < n) len[threadIdx.x] = load_caption(seqs, (long)img * n + threadIdx.x, T, false, tok[threadIdx.x]);
    if (threadIdx.x < n * CIDER_N) correct[threadIdx.x / CIDER_N][threadIdx.x % CIDER_N] = 0;
    if (threadIdx.x < 2) distinct[threadIdx.x] = 0;
    if (threadIdx.x == 0) words = 0;
    __syncthreads();
    if (threadIdx.x == 0) {
        int s = 0;
        for (int c = 0; c < n; ++c) s += len[c];
        words = s;
    }
    // distinct uni- and bigrams over the image: an item counts when no earlier caption or position holds the same n-gram
    for (int it = threadIdx.x; it < 2 * n * CIDER_MAXL; it += blockDim.x) {
        const int g = it / (n * CIDER_MAXL) + 1, c = (it / CIDER_MAXL) % n, p = it % CIDER_MAXL;
        if (p + g > len[c]) continue;
        bool first = true;
        for (int c2 = 0; c2 <= c && first; ++c2) {
            const int lim = c2 == c ? p : len[c2] - g + 1;
            for (int q = 0; q < lim; ++q) if (same_gram(tok[c] + p, tok[c2] + q, g)) { first = false; break; }
        }
        if (first) atomicAdd(&distinct[g - 1], 1);
    }
    // clipped n-gram counts of every caption against the image's other captions
    for (int it = threadIdx.x; it < n * CIDER_N * CIDER_MAXL; it += blockDim.x) {
        const int j = it / (CIDER_N * CIDER_MAXL), g = (it / CIDER_MAXL) % CIDER_N + 1, p = it % CIDER_MAXL;
        const int* h = tok[j];
        if (p + g > len[j]) continue;
        bool first = true;
        int tf = 0;
        for (int q = 0; q + g <= len[j]; ++q) {
            if (same_gram(h + p, h + q, g)) {
                if (q < p) { first = false; break; }
                ++tf;
            }
        }
        if (!first) continue;
        int max_ref = 0;
        for (int c = 0; c < n; ++c) {
            if (c == j) continue;
            int cnt = 0;
            for (int q = 0; q + g <= len[c]; ++q) cnt += same_gram(h + p, tok[c] + q, g) ? 1 : 0;
            max_ref = cnt > max_ref ? cnt : max_ref;
        }
        atomicAdd(&correct[j][g - 1], tf < max_ref ? tf : max_ref);
    }
    __syncthreads();
    if (threadIdx.x < 2) {
        const double d = (double)distinct[threadIdx.x] / (1e-6 + (double)words);
        (threadIdx.x == 0 ? out_div1 : out_div2)[img] = d;
    }
    if (threadIdx.x < n) {
        const int j = threadIdx.x, hl = len[j];
        int best = -1, best_diff = 0;
        for (int c = 0; c < n; ++c) {
            if (c == j) continue;
            const int d = abs(len[c] - hl);
            if (best < 0 || d < best_diff || (d == best_diff && len[c] < best)) { best = len[c]; best_diff = d; }
        }
        double b = 1.0;
        for (int k = 0; k < 2; ++k) {
            const int guess = hl - k > 0 ? hl - k : 0;
            b *= ((double)correct[j][k] + 1e-15) / ((double)guess + 1e-9);
        }
        b = pow(b, 0.5);
        const double ratio = ((double)hl + 1e-15) / ((double)best + 1e-9);
        if (ratio < 1.0) b *= exp(1.0 - 1.0 / ratio);
        out_bleu2[(long)img * n + j] = b;
        int* st = stats + ((long)img * n + j) * DIV_BLEU_STATS;
        for (int k = 0; k < CIDER_N; ++k) st[k] = correct[j][k];
        st[4] = hl;
        st[5] = best;
    }
}

// Corpus BLEU-1..4 of leave-one-out round j (one CTA per round): Bleu(4).compute_score over the images with caption j as the hypothesis,
// from the integer totals of correct and guessed n-grams and of hypothesis and closest reference lengths (bleu_scorer.py:226-260).
__global__ void __launch_bounds__(DIV_THREADS) mutual_bleu_kernel(const int* __restrict__ stats, int n_images, int n, double* __restrict__ out_mbleu) {
    __shared__ long long part[DIV_THREADS / 32][2 * CIDER_N + 2];
    const int j = blockIdx.x;
    long long acc[2 * CIDER_N + 2] = {};               // correct[4], guess[4], testlen, reflen
    for (int img = threadIdx.x; img < n_images; img += blockDim.x) {
        const int* st = stats + ((long)img * n + j) * DIV_BLEU_STATS;
        for (int k = 0; k < CIDER_N; ++k) {
            acc[k] += st[k];
            acc[CIDER_N + k] += st[4] - k > 0 ? st[4] - k : 0;
        }
        acc[2 * CIDER_N] += st[4];
        acc[2 * CIDER_N + 1] += st[5];
    }
    for (int f = 0; f < 2 * CIDER_N + 2; ++f) {
        long long v = acc[f];
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5][f] = v;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        long long tot[2 * CIDER_N + 2] = {};
        for (int wi = 0; wi < DIV_THREADS / 32; ++wi)
            for (int f = 0; f < 2 * CIDER_N + 2; ++f) tot[f] += part[wi][f];
        double b = 1.0, bleus[CIDER_N];
        for (int k = 0; k < CIDER_N; ++k) {
            b *= ((double)tot[k] + 1e-15) / ((double)tot[CIDER_N + k] + 1e-9);
            bleus[k] = pow(b, 1.0 / (k + 1));
        }
        const double ratio = ((double)tot[2 * CIDER_N] + 1e-15) / ((double)tot[2 * CIDER_N + 1] + 1e-9);
        for (int k = 0; k < CIDER_N; ++k) out_mbleu[j * CIDER_N + k] = ratio < 1.0 ? bleus[k] * exp(1.0 - 1.0 / ratio) : bleus[k];
    }
}

// gDiv-1 (compute_global_div_n with n = 1): distinct words over every caption, one CTA with a shared bitmap over the V + 1 ids.  A word
// outside [1, V] makes the count -1.
__global__ void __launch_bounds__(1024) global_div1_kernel(const long long* __restrict__ seqs, long rows, int T, int V1, double* __restrict__ out_gdiv1) {
    extern __shared__ unsigned int bits[];
    __shared__ int bad;
    __shared__ unsigned long long count;
    const int words = (V1 + 31) / 32;
    for (int i = threadIdx.x; i < words; i += blockDim.x) bits[i] = 0u;
    if (threadIdx.x == 0) { bad = 0; count = 0ull; }
    __syncthreads();
    const int cols = T < CIDER_MAXL ? T : CIDER_MAXL;
    for (long r = threadIdx.x; r < rows; r += blockDim.x) {
        for (int j = 0; j < cols; ++j) {
            const long long v = seqs[r * T + j];
            if (v == 0) break;
            if (v < 0 || v >= V1) { bad = 1; break; }
            atomicOr(&bits[v >> 5], 1u << (v & 31));
        }
    }
    __syncthreads();
    unsigned long long c = 0;
    for (int i = threadIdx.x; i < words; i += blockDim.x) c += __popc(bits[i]);
    atomicAdd(&count, c);
    __syncthreads();
    if (threadIdx.x == 0) *out_gdiv1 = bad ? -1.0 : (double)count;
}

size_t self_cider_smem(int n) {
    return (size_t)n * CIDER_N * CIDER_MAXL * sizeof(double) + (size_t)n * CIDER_N * sizeof(double) +
           (size_t)n * CIDER_N * CIDER_MAXL * sizeof(int) + (size_t)n * CIDER_MAXL * sizeof(int) + (size_t)n * sizeof(int);
}

int check_div_shapes(int n_images, int n, int T) {
    CAPB_REQUIRE(n_images >= 0, "negative image count");
    CAPB_REQUIRE(n >= 2 && n <= DIV_MAXN, "between 2 and 32 captions per image");
    CAPB_REQUIRE(T >= 1 && T <= CIDER_MAXL, "caption length between 1 and 64 tokens");
    return 0;
}

}  // namespace

int self_cider_div_launch(const double* mat, int n_images, int n, double* out_score, cudaStream_t stream) {
    CAPB_REQUIRE(n_images >= 0 && n >= 2 && n <= DIV_MAXN, "between 2 and 32 captions per image");
    if (n_images == 0) return 0;
    self_cider_div_kernel<<<n_images, 32, 0, stream>>>(mat, n, out_score);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int self_cider_launch(const CiderTable* t, const long long* seqs, int n_images, int n, int T, bool with_eos, double* out_mat, double* out_score,
                      cudaStream_t stream) {
    CAPB_REQUIRE(t != nullptr, "CIDEr table not initialised (init_scorer)");
    CAPB_REQUIRE(!t->corpus, "self-CIDEr needs a document-frequency table with a reference length; a corpus table has none");
    if (check_div_shapes(n_images, n, T)) return 1;
    if (n_images == 0) return 0;
    const size_t smem = self_cider_smem(n);
    CAPB_CHECK_CUDA(cudaFuncSetAttribute(self_cider_matrix_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    self_cider_matrix_kernel<<<n_images, DIV_THREADS, smem, stream>>>(t->slots, t->mask, t->log_ref_len, seqs, n, T, with_eos ? 1 : 0, out_mat);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return self_cider_div_launch(out_mat, n_images, n, out_score, stream);
}

int div_stats_launch(const long long* seqs, int n_images, int n, int T, int V1, double* out_div1, double* out_div2, double* out_gdiv1,
                     double* out_mbleu, double* out_bleu2, int* out_stats, cudaStream_t stream) {
    if (check_div_shapes(n_images, n, T)) return 1;
    CAPB_REQUIRE(V1 >= 2 && V1 <= (1 << 20), "V + 1 between 2 and 1 048 576");
    CAPB_REQUIRE(n_images > 0, "no images");
    const size_t bitmap = (size_t)((V1 + 31) / 32) * sizeof(unsigned int);
    CAPB_CHECK_CUDA(cudaFuncSetAttribute(global_div1_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bitmap));
    global_div1_kernel<<<1, 1024, bitmap, stream>>>(seqs, (long)n_images * n, T, V1, out_gdiv1);
    CAPB_CHECK_CUDA(cudaGetLastError());
    div_stats_kernel<<<n_images, DIV_THREADS, 0, stream>>>(seqs, n, T, out_div1, out_div2, out_bleu2, out_stats);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return corpus_bleu_launch(out_stats, n_images, n, out_mbleu, stream);
}

int corpus_bleu_launch(const int* stats, int n_images, int n, double* out_bleu, cudaStream_t stream) {
    mutual_bleu_kernel<<<n, DIV_THREADS, 0, stream>>>(stats, n_images, n, out_bleu);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace capb200

using namespace capb200;

extern "C" {

int capb200_self_cider(const capb200_cider_table* t, const long long* seqs, int n_images, int n, int T, int with_eos, double* out_mat,
                       double* out_score, void* stream) {
    CAPB_REQUIRE(t != nullptr && seqs && out_mat && out_score, "null argument");
    return self_cider_launch(t->t, seqs, n_images, n, T, with_eos != 0, out_mat, out_score, static_cast<cudaStream_t>(stream));
}

int capb200_self_cider_div(const double* mat, int n_images, int n, double* out_score, void* stream) {
    CAPB_REQUIRE(mat && out_score, "null argument");
    return self_cider_div_launch(mat, n_images, n, out_score, static_cast<cudaStream_t>(stream));
}

int capb200_div_stats(const long long* seqs, int n_images, int n, int T, int V1, double* out_div1, double* out_div2, double* out_gdiv1,
                      double* out_mbleu, double* out_bleu2, int* out_bleu_stats, void* stream) {
    CAPB_REQUIRE(seqs && out_div1 && out_div2 && out_gdiv1 && out_mbleu && out_bleu2 && out_bleu_stats, "null argument");
    return div_stats_launch(seqs, n_images, n, T, V1, out_div1, out_div2, out_gdiv1, out_mbleu, out_bleu2, out_bleu_stats,
                            static_cast<cudaStream_t>(stream));
}

}  // extern "C"
