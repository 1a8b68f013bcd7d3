// Element-wise kernels of the Transformer training steps (TransformerModel._forward teacher forcing, TransformerModel.py:340-348, and the
// train-mode sampling pass of LossWrapper's sc branch, loss_wrapper.py:56-73, with their backward passes).
//
// Decoder activations are TIME-major: row = t * N + n (position t of sequence n).  The same buffers then serve both forms of the forward
// pass -- the teacher-forced pass touches all L * N rows per kernel, the sampling pass the N rows of one position per kernel -- and the
// backward pass is always batched.  Every dropout site is keyed (seed, site, t, n * cols + c) (dropout.cuh), so a mask does not depend on
// which form produced the activation; encoder activations [B*R, D] use t = 0.
#include "common.cuh"
#include "dropout.cuh"
#include "kernels.cuh"

namespace capb200 {

namespace {

inline int blocks_for(long n) {
    long b = (n + 255) / 256;
    return (int)(b > sm_count() * 16 ? sm_count() * 16 : (b < 1 ? 1 : b));
}

// x[r, :] = dropout(lut[tok[r]] * scale + pe[t0 + r / rps]);  Embeddings (TransformerModel.py:208-215) + PositionalEncoding (:217-235)
__global__ void embed_pe_dropout_kernel(int rows, int rps, int D, const int* __restrict__ tok, const float* __restrict__ lut, const float* __restrict__ pe, float scale,
                                        int t0, unsigned long long seed, uint32_t site, float p, float* __restrict__ x, long ld) {
    const long total = (long)rows * D;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int r = (int)(i / D), c = (int)(i % D);
        const int t = t0 + r / rps, n = r % rps;
        const float v = fmaf(__ldg(lut + (long)tok[r] * D + c), scale, __ldg(pe + (long)t * D + c));
        x[(long)r * ld + c] = v * drop_scale(seed, site, (uint32_t)t, (uint32_t)((long)n * D + c), p);
    }
}

// d lut[tok[r], :] += scale * mask * dx[r, :]
__global__ void embed_pe_backward_kernel(int rows, int rps, int D, const int* __restrict__ tok, float scale, int t0, unsigned long long seed, uint32_t site, float p,
                                         const float* __restrict__ dx, long ld, float* __restrict__ dlut) {
    const long total = (long)rows * D;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int r = (int)(i / D), c = (int)(i % D);
        const int t = t0 + r / rps, n = r % rps;
        const float g = dx[(long)r * ld + c] * scale * drop_scale(seed, site, (uint32_t)t, (uint32_t)((long)n * D + c), p);
        if (g != 0.f) atomicAdd(dlut + (long)tok[r] * D + c, g);
    }
}

// out = a + dropout(b)     SublayerConnection (TransformerModel.py:89-101): x + dropout(sublayer(norm(x)))
__global__ void add_dropout_rows_kernel(int rows, int rps, int cols, int t0, const float* __restrict__ a, long ld_a, const float* __restrict__ b, long ld_b,
                                        float* __restrict__ out, long ld_o, unsigned long long seed, uint32_t site, float p) {
    const long total = (long)rows * cols;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int r = (int)(i / cols), c = (int)(i % cols);
        const int t = t0 + r / rps, n = r % rps;
        out[(long)r * ld_o + c] = a[(long)r * ld_a + c] + b[(long)r * ld_b + c] * drop_scale(seed, site, (uint32_t)t, (uint32_t)((long)n * cols + c), p);
    }
}

// dst = src * mask (the gradient of a dropped branch), optional ReLU gate: relu_of != nullptr -> zero where relu_of <= 0
__global__ void dropout_rows_copy_kernel(int rows, int rps, int cols, int t0, const float* __restrict__ src, long ld_s, float* __restrict__ dst, long ld_d,
                                         unsigned long long seed, uint32_t site, float p, const float* __restrict__ relu_of, long ld_r) {
    const long total = (long)rows * cols;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int r = (int)(i / cols), c = (int)(i % cols);
        const int t = t0 + r / rps, n = r % rps;
        float v = src[(long)r * ld_s + c] * drop_scale(seed, site, (uint32_t)t, (uint32_t)((long)n * cols + c), p);
        if (relu_of != nullptr && relu_of[(long)r * ld_r + c] <= 0.f) v = 0.f;
        dst[(long)r * ld_d + c] = v;
    }
}

// h = dropout(relu(h)) in place     PositionwiseFeedForward (TransformerModel.py:197-206) between w_1 and w_2; att_embed's ReLU + Dropout
__global__ void relu_dropout_rows_kernel(int rows, int rps, int cols, int t0, float* __restrict__ h, long ld, unsigned long long seed, uint32_t site, float p) {
    const long total = (long)rows * cols;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int r = (int)(i / cols), c = (int)(i % cols);
        const int t = t0 + r / rps, n = r % rps;
        const float v = h[(long)r * ld + c];
        h[(long)r * ld + c] = v > 0.f ? v * drop_scale(seed, site, (uint32_t)t, (uint32_t)((long)n * cols + c), p) : 0.f;
    }
}

// time-major [L][N][D] <-> sequence-major [N][L][D] row permutation
__global__ void permute_rows_kernel(int L, int N, int D, const float* __restrict__ src, long ld_s, float* __restrict__ dst, long ld_d, int to_seq_major) {
    const long total = (long)L * N * D;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const long row = i / D;
        const int c = (int)(i % D);
        long tm, sm;
        if (to_seq_major) { tm = row; const int t = (int)(row / N), n = (int)(row % N); sm = (long)n * L + t; dst[sm * ld_d + c] = src[tm * ld_s + c]; }
        else { sm = row; const int n = (int)(row / L), t = (int)(row % L); tm = (long)t * N + n; dst[tm * ld_d + c] = src[sm * ld_s + c]; }
    }
}

// tok[t * N + n] = labels[n, t]  (int64 -> int32, time-major);  key_mask[n, t] = (t == 0 || labels[n, t] != 0)   (TransformerModel.py:323-325)
__global__ void load_tokens_tm_kernel(const long long* __restrict__ labels, long ld, int N, int L, int* __restrict__ tok, float* __restrict__ key_mask, long ld_m) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N * L) return;
    const int t = i / N, n = i % N;
    const long long v = labels[(long)n * ld + t];
    tok[i] = (int)v;
    if (key_mask != nullptr) key_mask[(long)n * ld_m + t] = (t == 0 || v != 0) ? 1.f : 0.f;
}

}  // namespace

#define LAUNCH_OK() do { CAPB_CHECK_CUDA(cudaGetLastError()); return 0; } while (0)

int embed_pe_dropout_launch(int rows, int rps, int D, const int* tok, const float* lut, const float* pe, float scale, int t0, unsigned long long seed, int site,
                            float p, float* x, long ld, cudaStream_t st) {
    if (rows <= 0) return 0;
    embed_pe_dropout_kernel<<<blocks_for((long)rows * D), 256, 0, st>>>(rows, rps, D, tok, lut, pe, scale, t0, seed, (uint32_t)site, p, x, ld);
    LAUNCH_OK();
}
int embed_pe_backward_launch(int rows, int rps, int D, const int* tok, float scale, int t0, unsigned long long seed, int site, float p, const float* dx, long ld,
                             float* dlut, cudaStream_t st) {
    if (rows <= 0) return 0;
    embed_pe_backward_kernel<<<blocks_for((long)rows * D), 256, 0, st>>>(rows, rps, D, tok, scale, t0, seed, (uint32_t)site, p, dx, ld, dlut);
    LAUNCH_OK();
}
int add_dropout_rows_launch(int rows, int rps, int cols, int t0, const float* a, long ld_a, const float* b, long ld_b, float* out, long ld_o, unsigned long long seed,
                            int site, float p, cudaStream_t st) {
    if (rows <= 0) return 0;
    add_dropout_rows_kernel<<<blocks_for((long)rows * cols), 256, 0, st>>>(rows, rps, cols, t0, a, ld_a, b, ld_b, out, ld_o, seed, (uint32_t)site, p);
    LAUNCH_OK();
}
int dropout_rows_copy_launch(int rows, int rps, int cols, int t0, const float* src, long ld_s, float* dst, long ld_d, unsigned long long seed, int site, float p,
                             const float* relu_of, long ld_r, cudaStream_t st) {
    if (rows <= 0) return 0;
    dropout_rows_copy_kernel<<<blocks_for((long)rows * cols), 256, 0, st>>>(rows, rps, cols, t0, src, ld_s, dst, ld_d, seed, (uint32_t)site, p, relu_of, ld_r);
    LAUNCH_OK();
}
int relu_dropout_rows_launch(int rows, int rps, int cols, int t0, float* h, long ld, unsigned long long seed, int site, float p, cudaStream_t st) {
    if (rows <= 0) return 0;
    relu_dropout_rows_kernel<<<blocks_for((long)rows * cols), 256, 0, st>>>(rows, rps, cols, t0, h, ld, seed, (uint32_t)site, p);
    LAUNCH_OK();
}
int permute_rows_launch(int L, int N, int D, const float* src, long ld_s, float* dst, long ld_d, int to_seq_major, cudaStream_t st) {
    if (L <= 0 || N <= 0) return 0;
    permute_rows_kernel<<<blocks_for((long)L * N * D), 256, 0, st>>>(L, N, D, src, ld_s, dst, ld_d, to_seq_major);
    LAUNCH_OK();
}
int load_tokens_tm_launch(const long long* labels, long ld, int N, int L, int* tok, float* key_mask, long ld_m, cudaStream_t st) {
    if (N <= 0 || L <= 0) return 0;
    load_tokens_tm_kernel<<<(N * L + 255) / 256, 256, 0, st>>>(labels, ld, N, L, tok, key_mask, ld_m);
    LAUNCH_OK();
}
CAPB_DEFINE_SALT_SETTER(dropout_salt_set_tfm)

}  // namespace capb200
