// fp32 CUDA-core GEMM (exact-arithmetic mode) and the fp32 -> split-fp16 plane conversion.
//
// Same contract as the wgmma kernel in gemm_tc.cu:  C[M,N] = sum_s A_s[M,K_s] * W_s[N,K_s]^T + bias (+row bias, ReLU)
// with K-segments so torch.cat'ed LSTM inputs (AttModel.py:626,632) are never materialised.  This mode keeps the
// reference's fp32 FFMA arithmetic (only the summation order differs from cuBLAS / MKL) and serves as the on-device
// cross-check of the tensor-core path and as the path for shapes the TMA layout rules exclude.
#include "common.cuh"

namespace capb200 {

namespace {

constexpr int SBM = 128, SBN = 128, SBK = 16;

struct SimtParams {
    const float* A[kMaxSeg];
    const float* W[kMaxSeg];
    long lda[kMaxSeg];
    long ldw[kMaxSeg];
    int K[kMaxSeg];
    int nseg;
    int M, N;
    GemmEpilogue epi;
};

// Load 4 consecutive k-values of one row (zero beyond the matrix), vectorised when the address allows it.
__device__ __forceinline__ float4 load_row4(const float* base, long ld, int row, int nrows, int k, int K, bool vec_ok) {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (row < nrows && k < K) {
        const float* p = base + (long)row * ld + k;
        if (vec_ok && k + 3 < K) {
            v = __ldg(reinterpret_cast<const float4*>(p));
        } else {
            v.x = __ldg(p);
            if (k + 1 < K) v.y = __ldg(p + 1);
            if (k + 2 < K) v.z = __ldg(p + 2);
            if (k + 3 < K) v.w = __ldg(p + 3);
        }
    }
    return v;
}

__global__ void __launch_bounds__(256, 2) gemm_simt_kernel(const SimtParams p) {
    __shared__ __align__(16) float As[2][SBK][SBM + 4];
    __shared__ __align__(16) float Ws[2][SBK][SBN + 4];
    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;
    const int m0 = blockIdx.y * SBM, n0 = blockIdx.x * SBN;
    // global -> smem mapping: 128 rows x 16 k = 512 float4; each thread moves rows (tid>>2) and (tid>>2)+64, k-quad (tid&3)
    const int lrow = tid >> 2, lk = (tid & 3) * 4;

    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

    int buf = 0;
    for (int s = 0; s < p.nseg; ++s) {
        const float* A = p.A[s];
        const float* W = p.W[s];
        const long lda = p.lda[s], ldw = p.ldw[s];
        const int K = p.K[s];
        const bool va = ((lda & 3) == 0) && ((reinterpret_cast<uintptr_t>(A) & 15) == 0);
        const bool vw = ((ldw & 3) == 0) && ((reinterpret_cast<uintptr_t>(W) & 15) == 0);
        const int ktiles = (K + SBK - 1) / SBK;
        float4 ra0 = load_row4(A, lda, m0 + lrow, p.M, lk, K, va);
        float4 ra1 = load_row4(A, lda, m0 + lrow + 64, p.M, lk, K, va);
        float4 rw0 = load_row4(W, ldw, n0 + lrow, p.N, lk, K, vw);
        float4 rw1 = load_row4(W, ldw, n0 + lrow + 64, p.N, lk, K, vw);
        for (int kt = 0; kt < ktiles; ++kt) {
            // Two buffers + the barrier below are enough: a thread only gets here after the previous tile's barrier, and
            // every thread passes that barrier after finishing the tile that last read this buffer.
            As[buf][lk + 0][lrow] = ra0.x; As[buf][lk + 1][lrow] = ra0.y; As[buf][lk + 2][lrow] = ra0.z; As[buf][lk + 3][lrow] = ra0.w;
            As[buf][lk + 0][lrow + 64] = ra1.x; As[buf][lk + 1][lrow + 64] = ra1.y; As[buf][lk + 2][lrow + 64] = ra1.z; As[buf][lk + 3][lrow + 64] = ra1.w;
            Ws[buf][lk + 0][lrow] = rw0.x; Ws[buf][lk + 1][lrow] = rw0.y; Ws[buf][lk + 2][lrow] = rw0.z; Ws[buf][lk + 3][lrow] = rw0.w;
            Ws[buf][lk + 0][lrow + 64] = rw1.x; Ws[buf][lk + 1][lrow + 64] = rw1.y; Ws[buf][lk + 2][lrow + 64] = rw1.z; Ws[buf][lk + 3][lrow + 64] = rw1.w;
            __syncthreads();
            if (kt + 1 < ktiles) {
                const int k = (kt + 1) * SBK + lk;
                ra0 = load_row4(A, lda, m0 + lrow, p.M, k, K, va);
                ra1 = load_row4(A, lda, m0 + lrow + 64, p.M, k, K, va);
                rw0 = load_row4(W, ldw, n0 + lrow, p.N, k, K, vw);
                rw1 = load_row4(W, ldw, n0 + lrow + 64, p.N, k, K, vw);
            }
#pragma unroll
            for (int k = 0; k < SBK; ++k) {
                const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
                const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][64 + ty * 4]);
                const float4 b0 = *reinterpret_cast<const float4*>(&Ws[buf][k][tx * 4]);
                const float4 b1 = *reinterpret_cast<const float4*>(&Ws[buf][k][64 + tx * 4]);
                const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
                const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
                for (int i = 0; i < 8; ++i)
#pragma unroll
                    for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
            }
            buf ^= 1;
        }
    }

    const GemmEpilogue& e = p.epi;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int row = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
        if (row >= p.M) continue;
        const float* rb = e.row_bias ? e.row_bias + (long)(row / e.rows_per_group) * e.ld_row_bias : nullptr;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int col = n0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + (j - 4));
            if (col >= p.N) continue;
            float x = acc[i][j];
            if (e.bias) x += __ldg(e.bias + col);
            if (rb) x += __ldg(rb + col);
            if (e.residual) x += e.residual[(long)row * e.ld_res + col];
            if (e.relu) x = fmaxf(x, 0.f);
            if (e.C) e.C[(long)row * e.ldc + col] = x;
            if (e.C_hi) {
                __half h, l;
                split_f32(x, h, l);
                e.C_hi[(long)row * e.ldcs + col] = h;
                e.C_lo[(long)row * e.ldcs + col] = l;
            }
        }
    }
}

// Both conversion kernels also enforce the one numeric precondition of the split-fp16 scheme: |x| < 65504 and finite (fp16 range).  A
// violation sets the process-wide flag (pinned, host-mapped) that every C-ABI entry point reports as an error (range_flag_*).
__global__ void split_planes_kernel(const float* __restrict__ x, long ldx, int rows, int cols, __half* __restrict__ hi,
                                    __half* __restrict__ lo, long ldh, int* __restrict__ range_flag) {
    const long total = (long)rows * cols;
    bool bad = false;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int r = (int)(i / cols), c = (int)(i % cols);
        __half h, l;
        const float v = __ldg(x + (long)r * ldx + c);
        bad |= !(fabsf(v) < 65504.0f);
        split_f32(v, h, l);
        hi[(long)r * ldh + c] = h;
        lo[(long)r * ldh + c] = l;
    }
    if (bad && range_flag != nullptr) *range_flag = 1;
}

// 128-bit variant for 16-byte aligned rows (the 75.5 MB bottom-up feature tile of every decode goes through here): one float4 in, two 8-byte
// stores out per thread and no integer division per element.
__global__ void split_planes_vec4_kernel(const float* __restrict__ x, long ldx, int rows, int cols4, __half* __restrict__ hi, __half* __restrict__ lo,
                                         long ldh, int* __restrict__ range_flag) {
    const long total = (long)rows * cols4;
    bool bad = false;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const long r = i / cols4;
        const int c = (int)(i - r * cols4) * 4;
        const float4 v = __ldg(reinterpret_cast<const float4*>(x + r * ldx + c));
        bad |= !(fabsf(v.x) < 65504.0f) || !(fabsf(v.y) < 65504.0f) || !(fabsf(v.z) < 65504.0f) || !(fabsf(v.w) < 65504.0f);
        __align__(8) __half h[4];
        __align__(8) __half l[4];
        split_f32(v.x, h[0], l[0]); split_f32(v.y, h[1], l[1]); split_f32(v.z, h[2], l[2]); split_f32(v.w, h[3], l[3]);
        *reinterpret_cast<uint2*>(hi + r * ldh + c) = *reinterpret_cast<const uint2*>(h);
        *reinterpret_cast<uint2*>(lo + r * ldh + c) = *reinterpret_cast<const uint2*>(l);
    }
    if (bad && range_flag != nullptr) *range_flag = 1;
}

__global__ void split_planes_interleave_kernel(const float* __restrict__ x, long ldx, int H, int cols, __half* __restrict__ hi,
                                               __half* __restrict__ lo, long ldh, int* __restrict__ range_flag) {
    const long total = (long)4 * H * cols;
    bool bad = false;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int rd = (int)(i / cols), c = (int)(i % cols);          // destination row 4*j+g
        const int j = rd >> 2, g = rd & 3;
        __half h, l;
        const float v = __ldg(x + (long)(g * H + j) * ldx + c);
        bad |= !(fabsf(v) < 65504.0f);
        split_f32(v, h, l);
        hi[(long)rd * ldh + c] = h;
        lo[(long)rd * ldh + c] = l;
    }
    if (bad && range_flag != nullptr) *range_flag = 1;
}

}  // namespace

// Process-wide "a value outside the fp16 range reached a split-fp16 conversion" flag: one int in pinned, host-mapped, portable memory
// (kernels on any device write it through the unified address; the host reads it without a copy once the writing stream has been
// synchronised by whoever consumes the results).
static int* g_range_flag = nullptr;
int* range_flag_ptr() {
    static std::atomic<int> once{0};
    int expected = 0;
    if (g_range_flag == nullptr && once.compare_exchange_strong(expected, 1)) {
        int* p = nullptr;
        if (cudaHostAlloc(&p, sizeof(int), cudaHostAllocMapped | cudaHostAllocPortable) == cudaSuccess) { *p = 0; g_range_flag = p; }
        else (void)cudaGetLastError();
    }
    return g_range_flag;
}
int range_flag_read(int reset) {
    int* p = range_flag_ptr();
    if (p == nullptr) return 0;
    const int v = *reinterpret_cast<volatile int*>(p);
    if (reset) *reinterpret_cast<volatile int*>(p) = 0;
    return v;
}

int split_planes_interleave_launch(const float* x, long ldx, int H, int cols, __half* hi, __half* lo, long ldh, cudaStream_t stream) {
    const long total = (long)4 * H * cols;
    if (total <= 0) return 0;
    int blocks = (int)((total + 255) / 256);
    if (blocks > sm_count() * 16) blocks = sm_count() * 16;
    split_planes_interleave_kernel<<<blocks, 256, 0, stream>>>(x, ldx, H, cols, hi, lo, ldh, range_flag_ptr());
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int gemm_simt_launch(const GemmProblem& g, cudaStream_t stream) {
    CAPB_REQUIRE(g.nseg >= 1 && g.nseg <= kMaxSeg, "1..3 K-segments");
    CAPB_REQUIRE(g.epi.lstm == 0, "the fused LSTM epilogue exists on the tensor-core path only");
    if (g.M <= 0 || g.N <= 0) return 0;
    SimtParams p;
    memset(&p, 0, sizeof(p));
    p.nseg = g.nseg;
    p.M = g.M;
    p.N = g.N;
    for (int s = 0; s < g.nseg; ++s) {
        CAPB_REQUIRE(g.seg[s].A != nullptr && g.seg[s].W != nullptr, "fp32 operands required in SIMT mode");
        p.A[s] = g.seg[s].A; p.W[s] = g.seg[s].W;
        p.lda[s] = g.seg[s].lda; p.ldw[s] = g.seg[s].ldw; p.K[s] = g.seg[s].K;
    }
    p.epi = g.epi;
    if (p.epi.rows_per_group < 1) p.epi.rows_per_group = 1;
    dim3 grid(cdiv(g.N, SBN), cdiv(g.M, SBM));
    gemm_simt_kernel<<<grid, 256, 0, stream>>>(p);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int split_planes_launch(const float* x, long ldx, int rows, int cols, __half* hi, __half* lo, long ldh, cudaStream_t stream) {
    if (rows <= 0 || cols <= 0) return 0;
    const long total = (long)rows * cols;
    const bool vec = (cols & 3) == 0 && (ldx & 3) == 0 && (ldh & 3) == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(hi) & 7) == 0 && (reinterpret_cast<uintptr_t>(lo) & 7) == 0;
    if (vec) {
        int vb = (int)((total / 4 + 255) / 256);
        if (vb > sm_count() * 16) vb = sm_count() * 16;
        split_planes_vec4_kernel<<<vb, 256, 0, stream>>>(x, ldx, rows, cols / 4, hi, lo, ldh, range_flag_ptr());
        CAPB_CHECK_CUDA(cudaGetLastError());
        return 0;
    }
    int blocks = (int)((total + 255) / 256);
    if (blocks > sm_count() * 16) blocks = sm_count() * 16;
    split_planes_kernel<<<blocks, 256, 0, stream>>>(x, ldx, rows, cols, hi, lo, ldh, range_flag_ptr());
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace capb200
