// Generic fp32 CUDA-core GEMM for the SCST backward pass:  C[M,N] = op(A)[M,K] * op(B)[K,N] (+ C if accumulate)
//
//   TA = 0: A stored [M, K] (pitch lda)      TA = 1: A stored [K, M]   (dW = dY^T * X reads dY this way)
//   TB = 0: B stored [K, N] (pitch ldb)      TB = 1: B stored [N, K]   (nn.Linear forward: x * W^T)
// The training shapes are skinny (M = B * sample_n = 50..60 rows, or K = T * rows ~ 1000 for the weight gradients), i.e. weight-
// streaming bound; 64x64x16 tiles with 4x4 register blocks keep enough CTAs in flight for those shapes.
#include <cstring>

#include "common.cuh"
#include "kernels.cuh"

namespace capb200 {

namespace {

constexpr int GT = 64, GK = 16;

template <int TA, int TB>
__global__ void __launch_bounds__(256) gemm_generic_kernel(int M, int N, int K, const float* __restrict__ A, long lda, const float* __restrict__ B,
                                                           long ldb, float* __restrict__ C, long ldc, int accumulate, const float* __restrict__ bias) {
    __shared__ float As[GK][GT + 1];
    __shared__ float Bs[GK][GT + 1];
    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;
    const int m0 = blockIdx.y * GT, n0 = blockIdx.x * GT;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    for (int k0 = 0; k0 < K; k0 += GK) {
        // 64 x 16 elements per operand tile, 4 per thread
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int idx = tid + 256 * u;
            int mm, kk;
            if (TA) { mm = idx & 63; kk = idx >> 6; } else { kk = idx & 15; mm = idx >> 4; }       // contiguous index follows the storage order
            float v = 0.f;
            if (m0 + mm < M && k0 + kk < K) v = TA ? A[(long)(k0 + kk) * lda + m0 + mm] : A[(long)(m0 + mm) * lda + k0 + kk];
            As[kk][mm] = v;
            int nn, kb;
            if (TB) { kb = idx & 15; nn = idx >> 4; } else { nn = idx & 63; kb = idx >> 6; }
            float w = 0.f;
            if (n0 + nn < N && k0 + kb < K) w = TB ? B[(long)(n0 + nn) * ldb + k0 + kb] : B[(long)(k0 + kb) * ldb + n0 + nn];
            Bs[kb][nn] = w;
        }
        __syncthreads();
        // each K-tile is summed on its own and then added to the running total: a weight gradient's K ~ 1000 rows would otherwise run
        // through one fp32 accumulator whose rounding grows with the running sum at every step (K / GK additions to it instead of K)
        float part[4][4];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) part[i][j] = 0.f;
#pragma unroll
        for (int k = 0; k < GK; ++k) {
            float a[4], b[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) a[i] = As[k][ty * 4 + i];
#pragma unroll
            for (int j = 0; j < 4; ++j) b[j] = Bs[k][tx * 4 + j];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) part[i][j] = fmaf(a[i], b[j], part[i][j]);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] += part[i][j];
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int row = m0 + ty * 4 + i;
        if (row >= M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int col = n0 + tx * 4 + j;
            if (col >= N) continue;
            float v = acc[i][j];
            if (bias != nullptr) v += bias[col];
            float* c = C + (long)row * ldc + col;
            *c = accumulate ? (*c + v) : v;
        }
    }
}

// column sums: out[c] (+)= sum_r x[r, c]   (bias gradients).  Block = 32 columns x 8 row groups: every warp reads 128-byte row segments, the eight
// groups walk disjoint rows four loads at a time and meet in shared memory (a single thread per column walking ~1000 rows was latency bound).
__global__ void __launch_bounds__(256) colsum_kernel(int rows, int cols, const float* __restrict__ x, long ld, float* __restrict__ out, int accumulate) {
    __shared__ float sh[8][33];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + tx;
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
    if (c < cols) {
        int r = ty;
        for (; r + 24 < rows; r += 32) {
            s0 += x[(long)r * ld + c]; s1 += x[(long)(r + 8) * ld + c]; s2 += x[(long)(r + 16) * ld + c]; s3 += x[(long)(r + 24) * ld + c];
        }
        for (; r < rows; r += 8) s0 += x[(long)r * ld + c];
    }
    sh[ty][tx] = (s0 + s1) + (s2 + s3);
    __syncthreads();
    if (ty == 0 && c < cols) {
        float s = 0.f;
#pragma unroll
        for (int g = 0; g < 8; ++g) s += sh[g][tx];
        out[c] = accumulate ? out[c] + s : s;
    }
}

}  // namespace

int gemm_generic_launch(int ta, int tb, int M, int N, int K, const float* A, long lda, const float* B, long ldb, float* C, long ldc, int accumulate,
                        const float* bias, cudaStream_t st) {
    if (M <= 0 || N <= 0) return 0;
    dim3 grid(cdiv(N, GT), cdiv(M, GT));
    if (!ta && !tb) gemm_generic_kernel<0, 0><<<grid, 256, 0, st>>>(M, N, K, A, lda, B, ldb, C, ldc, accumulate, bias);
    else if (!ta && tb) gemm_generic_kernel<0, 1><<<grid, 256, 0, st>>>(M, N, K, A, lda, B, ldb, C, ldc, accumulate, bias);
    else if (ta && !tb) gemm_generic_kernel<1, 0><<<grid, 256, 0, st>>>(M, N, K, A, lda, B, ldb, C, ldc, accumulate, bias);
    else gemm_generic_kernel<1, 1><<<grid, 256, 0, st>>>(M, N, K, A, lda, B, ldb, C, ldc, accumulate, bias);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int colsum_launch(int rows, int cols, const float* x, long ld, float* out, int accumulate, cudaStream_t st) {
    if (cols <= 0) return 0;
    colsum_kernel<<<cdiv(cols, 32), 256, 0, st>>>(rows, cols, x, ld, out, accumulate);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace capb200

// ---------------------------------------------------------------------------------------------------------------------
// Skinny split-K GEMM for the training step:  C[M,N] (+)= sum_s A_s[M,K_s] * op(B_s)  (+ bias[N] + row_bias[row / rpg, N])
// M = B * sample_n is 50..60 rows, so a conventional tiling leaves most SMs idle while one CTA walks a 3000-deep K; here the K-steps of
// all segments are split across blockIdx.y so ~2 CTAs per SM stream disjoint slices of the weights, and a second pass adds the partial
// sums in a fixed order (deterministic, no atomics).
// ---------------------------------------------------------------------------------------------------------------------
namespace capb200 {

namespace {

struct SkinnyParams {
    const float* A[3];
    const float* B[3];
    long lda[3], ldb[3];
    int K[3], tb[3];
    int nseg, M, N, ksteps_total, ksplit;
    float* out;          // C (ksplit == 1) or the partial buffer [ksplit][M][N]
    long ldo;
    const float* bias;
    const float* row_bias;
    long ld_rb;
    int rpg, accumulate;
};

__global__ void __launch_bounds__(256) gemm_skinny_kernel(const SkinnyParams p) {
    __shared__ float As[GK][GT + 1];
    __shared__ float Bs[GK][GT + 1];
    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;
    const int n0 = blockIdx.x * GT, m0 = blockIdx.z * GT;
    const int per = (p.ksteps_total + p.ksplit - 1) / p.ksplit;
    const int ks0 = blockIdx.y * per, ks1 = min(p.ksteps_total, ks0 + per);
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    int seg = 0, seg_first = 0;
    for (int ks = ks0; ks < ks1; ++ks) {
        while (seg < p.nseg - 1 && ks >= seg_first + (p.K[seg] + GK - 1) / GK) { seg_first += (p.K[seg] + GK - 1) / GK; ++seg; }
        const int k0 = (ks - seg_first) * GK;
        const int K = p.K[seg];
        const float* A = p.A[seg];
        const float* B = p.B[seg];
        const long lda = p.lda[seg], ldb = p.ldb[seg];
        const int tb = p.tb[seg];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int idx = tid + 256 * u;
            const int kk = idx & 15, mm = idx >> 4;
            As[kk][mm] = (m0 + mm < p.M && k0 + kk < K) ? A[(long)(m0 + mm) * lda + k0 + kk] : 0.f;
            int nn, kb;
            if (tb) { kb = idx & 15; nn = idx >> 4; } else { nn = idx & 63; kb = idx >> 6; }
            float w = 0.f;
            if (n0 + nn < p.N && k0 + kb < K) w = tb ? B[(long)(n0 + nn) * ldb + k0 + kb] : B[(long)(k0 + kb) * ldb + n0 + nn];
            Bs[kb][nn] = w;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < GK; ++k) {
            float a[4], b[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) a[i] = As[k][ty * 4 + i];
#pragma unroll
            for (int j = 0; j < 4; ++j) b[j] = Bs[k][tx * 4 + j];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int row = m0 + ty * 4 + i;
        if (row >= p.M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int col = n0 + tx * 4 + j;
            if (col >= p.N) continue;
            float v = acc[i][j];
            if (p.ksplit == 1) {
                if (p.bias) v += p.bias[col];
                if (p.row_bias) v += p.row_bias[(long)(row / p.rpg) * p.ld_rb + col];
                float* c = p.out + (long)row * p.ldo + col;
                *c = p.accumulate ? (*c + v) : v;
            } else {
                p.out[((long)blockIdx.y * p.M + row) * p.N + col] = v;
            }
        }
    }
}

// Same problem on the tensor cores: 3xTF32 (hi*lo + lo*hi + hi*hi, fp32 accumulate) through mma.sync.m16n8k8, reading the fp32 weights
// as they are (no repack after optimizer steps; TF32 keeps the fp32 exponent, so small gradients do not underflow the way fp16 planes
// would).  The shapes are weight-streaming bound, so the legacy mma path is enough; tile 64 x 64 x 32, 8 warps as 2 (M) x 4 (N).
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hi) : "f"(x));
    const float r = x - __uint_as_float(hi);
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lo) : "f"(r));
}
__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// One 16-deep K-slice per thread in flight (two float4 loads) would cap a weight-streaming GEMM at ~1 TB/s, so raw fp32 tiles are
// staged with cp.async through a 4-stage ring of 32-deep K-slices (18 KB per stage, 3 CTAs per SM => ~160 KB of loads in flight per SM);
// the TF32 hi/lo split happens on the fragments.
constexpr int S2_BK = 32, S2_STAGES = 4;
constexpr int S2_ALD = S2_BK + 4;        // A / B^T rows: 36 floats (16-byte multiples, conflict-free fragment loads)
constexpr int S2_BLD = GT + 8;           // B rows [k][n]: 72 floats
constexpr int S2_STAGE_FLOATS = GT * S2_ALD + GT * S2_ALD;     // A tile + B tile (TB: 64 x 36; else 32 x 72 = the same 2304 floats)

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc, int src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gsrc), "r"(src_bytes) : "memory");
}

// TA = 1: A stored [K, M] (the dY operand of a weight gradient dW = dY^T X): its tile is staged as [k][m] rows like a [K, N] W tile.
template <int TB, int TA>
__global__ void __launch_bounds__(256) gemm_skinny_tf32_v2_kernel(const SkinnyParams p) {
    extern __shared__ __align__(16) float s2[];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int g = lane >> 2, tig = lane & 3;
    const int wm = (warp >> 2) * 32, wn = (warp & 3) * 16;
    const int n0 = blockIdx.x * GT, m0 = blockIdx.z * GT;
    const int per = (p.ksteps_total + p.ksplit - 1) / p.ksplit;
    const int ks0 = blockIdx.y * per, ks1 = min(p.ksteps_total, ks0 + per);
    const int nsteps = ks1 > ks0 ? ks1 - ks0 : 0;
    float acc[2][2][4];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[i][j][q] = 0.f;

    // issue the loads of K-step `ks` (global index) into ring slot `slot`
    auto issue = [&](int ks, int slot) {
        int seg = 0, first = 0;
        while (seg < p.nseg - 1 && ks >= first + (p.K[seg] + S2_BK - 1) / S2_BK) { first += (p.K[seg] + S2_BK - 1) / S2_BK; ++seg; }
        const int k0 = (ks - first) * S2_BK, K = p.K[seg];
        float* As = s2 + slot * S2_STAGE_FLOATS;
        float* Bs = As + GT * S2_ALD;
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            const int idx = tid + 256 * u;                  // 512 float4 per operand tile
            if (TA) {   // A stored [K, M]: 32 rows (k) x 16 float4 (m)
                const int row = idx >> 4, mq = (idx & 15) * 4;
                const bool ok = (k0 + row < K) && (m0 + mq < p.M);
                const float* src = ok ? p.A[seg] + (long)(k0 + row) * p.lda[seg] + m0 + mq : p.A[seg];
                cp_async16(As + row * S2_BLD + mq, src, ok ? 16 : 0);
            } else {    // A tile: 64 rows x 8 float4
                const int row = idx >> 3, kq = (idx & 7) * 4;
                const bool ok = (m0 + row < p.M) && (k0 + kq < K);
                const float* src = ok ? p.A[seg] + (long)(m0 + row) * p.lda[seg] + k0 + kq : p.A[seg];
                cp_async16(As + row * S2_ALD + kq, src, ok ? 16 : 0);
            }
            if (TB) {   // W stored [N, K]: 64 rows (n) x 8 float4 (k)
                const int row = idx >> 3, kq = (idx & 7) * 4;
                const bool ok = (n0 + row < p.N) && (k0 + kq < K);
                const float* src = ok ? p.B[seg] + (long)(n0 + row) * p.ldb[seg] + k0 + kq : p.B[seg];
                cp_async16(Bs + row * S2_ALD + kq, src, ok ? 16 : 0);
            } else {    // W stored [K, N]: 32 rows (k) x 16 float4 (n)
                const int row = idx >> 4, nq = (idx & 15) * 4;
                const bool ok = (k0 + row < K) && (n0 + nq < p.N);
                const float* src = ok ? p.B[seg] + (long)(k0 + row) * p.ldb[seg] + n0 + nq : p.B[seg];
                cp_async16(Bs + row * S2_BLD + nq, src, ok ? 16 : 0);
            }
        }
    };
#pragma unroll
    for (int s = 0; s < S2_STAGES - 1; ++s) {
        if (s < nsteps) issue(ks0 + s, s);
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
    for (int it = 0; it < nsteps; ++it) {
        asm volatile("cp.async.wait_group %0;" ::"n"(S2_STAGES - 2) : "memory");
        __syncthreads();                                    // slot (it-1) % STAGES is free again, slot it % STAGES has landed
        if (it + S2_STAGES - 1 < nsteps) issue(ks0 + it + S2_STAGES - 1, (it + S2_STAGES - 1) % S2_STAGES);
        asm volatile("cp.async.commit_group;" ::: "memory");
        const float* As = s2 + (it % S2_STAGES) * S2_STAGE_FLOATS;
        const float* Bs = As + GT * S2_ALD;
#pragma unroll
        for (int kk = 0; kk < S2_BK; kk += 8) {
            uint32_t ah[2][4], al[2][4], bh[2][2], bl[2][2];
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int r = wm + i * 16 + g;
                if (TA) {
                    split_tf32(As[(kk + tig) * S2_BLD + r], ah[i][0], al[i][0]);
                    split_tf32(As[(kk + tig) * S2_BLD + r + 8], ah[i][1], al[i][1]);
                    split_tf32(As[(kk + tig + 4) * S2_BLD + r], ah[i][2], al[i][2]);
                    split_tf32(As[(kk + tig + 4) * S2_BLD + r + 8], ah[i][3], al[i][3]);
                } else {
                    split_tf32(As[r * S2_ALD + kk + tig], ah[i][0], al[i][0]);
                    split_tf32(As[(r + 8) * S2_ALD + kk + tig], ah[i][1], al[i][1]);
                    split_tf32(As[r * S2_ALD + kk + tig + 4], ah[i][2], al[i][2]);
                    split_tf32(As[(r + 8) * S2_ALD + kk + tig + 4], ah[i][3], al[i][3]);
                }
            }
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const int c = wn + j * 8 + g;
                if (TB) {
                    split_tf32(Bs[c * S2_ALD + kk + tig], bh[j][0], bl[j][0]);
                    split_tf32(Bs[c * S2_ALD + kk + tig + 4], bh[j][1], bl[j][1]);
                } else {
                    split_tf32(Bs[(kk + tig) * S2_BLD + c], bh[j][0], bl[j][0]);
                    split_tf32(Bs[(kk + tig + 4) * S2_BLD + c], bh[j][1], bl[j][1]);
                }
            }
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    mma_tf32(acc[i][j], ah[i], bl[j]);
                    mma_tf32(acc[i][j], al[i], bh[j]);
                    mma_tf32(acc[i][j], ah[i], bh[j]);
                }
        }
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int row = m0 + wm + i * 16 + g + (q >> 1) * 8;
                const int col = n0 + wn + j * 8 + 2 * tig + (q & 1);
                if (row >= p.M || col >= p.N) continue;
                float v = acc[i][j][q];
                if (p.ksplit == 1) {
                    if (p.bias) v += p.bias[col];
                    if (p.row_bias) v += p.row_bias[(long)(row / p.rpg) * p.ld_rb + col];
                    float* c = p.out + (long)row * p.ldo + col;
                    *c = p.accumulate ? (*c + v) : v;
                } else {
                    p.out[((long)blockIdx.y * p.M + row) * p.N + col] = v;
                }
            }
}

__global__ void skinny_reduce_kernel(int M, int N, int ksplit, const float* __restrict__ part, float* __restrict__ C, long ldc, const float* __restrict__ bias,
                                     const float* __restrict__ row_bias, long ld_rb, int rpg, int accumulate) {
    const long total = (long)M * N;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
        const int row = (int)(i / N), col = (int)(i % N);
        float v = 0.f;
        for (int s = 0; s < ksplit; ++s) v += part[(long)s * total + i];
        if (bias) v += bias[col];
        if (row_bias) v += row_bias[(long)(row / rpg) * ld_rb + col];
        float* c = C + (long)row * ldc + col;
        *c = accumulate ? (*c + v) : v;
    }
}

}  // namespace

int gemm_skinny_launch(int M, int N, int nseg, const float* const* A, const long* lda, const float* const* B, const long* ldb, const int* K, const int* tb,
                       float* C, long ldc, const float* bias, const float* row_bias, long ld_rb, int rpg, int accumulate, float* scratch,
                       size_t scratch_floats, int mode, cudaStream_t st) {
    if (M <= 0 || N <= 0) return 0;
    CAPB_REQUIRE(nseg >= 1 && nseg <= 3, "1..3 segments");
    SkinnyParams p;
    memset(&p, 0, sizeof(p));
    p.nseg = nseg; p.M = M; p.N = N;
    // the tensor-core kernel needs 16-byte aligned float4 rows and one storage order for all segments
    bool tc = (mode != 0);
    for (int s = 0; s < nseg; ++s) {
        tc = tc && tb[s] == tb[0] && K[s] % 4 == 0 && lda[s] % 4 == 0 && ldb[s] % 4 == 0 && (reinterpret_cast<uintptr_t>(A[s]) & 15) == 0 &&
             (reinterpret_cast<uintptr_t>(B[s]) & 15) == 0 && (tb[s] || N % 4 == 0);
    }
    const int bk = tc ? S2_BK : GK;
    int ksteps = 0;
    for (int s = 0; s < nseg; ++s) {
        p.A[s] = A[s]; p.B[s] = B[s]; p.lda[s] = lda[s]; p.ldb[s] = ldb[s]; p.K[s] = K[s]; p.tb[s] = tb[s];
        ksteps += cdiv(K[s], bk);
    }
    p.ksteps_total = ksteps;
    const int tiles = cdiv(N, GT) * cdiv(M, GT);
    int ksplit = ((tc ? 3 : 2) * sm_count() + tiles - 1) / tiles;          // CTAs resident per SM: 3 (tensor cores, 74 KB of shared memory each) or 2
    if (ksplit > ksteps / 4) ksplit = ksteps / 4;                  // at least 4 K-steps per CTA
    if (ksplit < 1) ksplit = 1;
    while (ksplit > 1 && (size_t)ksplit * M * N > scratch_floats) --ksplit;
    p.ksplit = ksplit;
    p.bias = bias; p.row_bias = row_bias; p.ld_rb = ld_rb; p.rpg = rpg < 1 ? 1 : rpg; p.accumulate = accumulate;
    if (ksplit == 1) { p.out = C; p.ldo = ldc; } else { p.out = scratch; p.ldo = N; }
    dim3 grid(cdiv(N, GT), ksplit, cdiv(M, GT));
    if (tc) {
        constexpr int smem = S2_STAGES * S2_STAGE_FLOATS * (int)sizeof(float);
        static std::atomic<unsigned long long> configured{0};
        if (first_use_on_device(configured)) {
            CAPB_CHECK_CUDA(cudaFuncSetAttribute(gemm_skinny_tf32_v2_kernel<0, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
            CAPB_CHECK_CUDA(cudaFuncSetAttribute(gemm_skinny_tf32_v2_kernel<1, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        }
        if (tb[0]) gemm_skinny_tf32_v2_kernel<1, 0><<<grid, 256, smem, st>>>(p);
        else gemm_skinny_tf32_v2_kernel<0, 0><<<grid, 256, smem, st>>>(p);
    } else {
        gemm_skinny_kernel<<<grid, 256, 0, st>>>(p);
    }
    CAPB_CHECK_CUDA(cudaGetLastError());
    if (ksplit > 1) {
        long blocks = ((long)M * N + 255) / 256;
        if (blocks > sm_count() * 8) blocks = sm_count() * 8;
        skinny_reduce_kernel<<<(int)blocks, 256, 0, st>>>(M, N, ksplit, scratch, C, ldc, bias, row_bias, ld_rb, p.rpg, accumulate);
        CAPB_CHECK_CUDA(cudaGetLastError());
    }
    return 0;
}

// Weight gradient on the tensor cores:  G[M, N] (+)= dY[K, M]^T * X[K, N]  (3xTF32, fp32 accumulate).  Falls back to the fp32 CUDA-core
// kernel when the operands are not 16-byte aligned or mode == 0.
int gemm_wgrad_launch(int M, int N, int K, const float* dY, long ld_dy, const float* X, long ld_x, float* G, long ld_g, int accumulate, int mode,
                      cudaStream_t st) {
    if (M <= 0 || N <= 0) return 0;
    const bool ok = mode != 0 && K > 0 && M % 4 == 0 && N % 4 == 0 && ld_dy % 4 == 0 && ld_x % 4 == 0 && (reinterpret_cast<uintptr_t>(dY) & 15) == 0 &&
                    (reinterpret_cast<uintptr_t>(X) & 15) == 0;
    if (!ok) return gemm_generic_launch(1, 0, M, N, K, dY, ld_dy, X, ld_x, G, ld_g, accumulate, nullptr, st);
    SkinnyParams p;
    memset(&p, 0, sizeof(p));
    p.nseg = 1; p.M = M; p.N = N;
    p.A[0] = dY; p.lda[0] = ld_dy; p.B[0] = X; p.ldb[0] = ld_x; p.K[0] = K; p.tb[0] = 0;
    p.ksteps_total = cdiv(K, S2_BK);
    p.ksplit = 1;
    p.out = G; p.ldo = ld_g; p.rpg = 1; p.accumulate = accumulate;
    constexpr int smem = S2_STAGES * S2_STAGE_FLOATS * (int)sizeof(float);
    static std::atomic<unsigned long long> configured{0};
    if (first_use_on_device(configured)) {
        CAPB_CHECK_CUDA(cudaFuncSetAttribute(gemm_skinny_tf32_v2_kernel<0, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    }
    dim3 grid(cdiv(N, GT), 1, cdiv(M, GT));
    gemm_skinny_tf32_v2_kernel<0, 1><<<grid, 256, smem, st>>>(p);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace capb200
