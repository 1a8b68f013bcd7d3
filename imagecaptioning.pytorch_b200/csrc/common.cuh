// Shared host/device helpers for the capb200 kernels.
#pragma once
#include <atomic>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

namespace capb200 {

// ---- error plumbing: every C-ABI entry point returns 0 or stores a message retrievable with capb200_last_error()
void set_error(const std::string& msg);
#define CAPB_CHECK_CUDA(expr)                                                                          \
    do {                                                                                               \
        cudaError_t _e = (expr);                                                                       \
        if (_e != cudaSuccess) {                                                                       \
            capb200::set_error(std::string(#expr) + " failed: " + cudaGetErrorString(_e) + " at " +    \
                               __FILE__ + ":" + std::to_string(__LINE__));                            \
            return 1;                                                                                  \
        }                                                                                              \
    } while (0)
#define CAPB_REQUIRE(cond, msg)                                                                        \
    do {                                                                                               \
        if (!(cond)) {                                                                                 \
            capb200::set_error(std::string("requirement failed: ") + #cond + " -- " + (msg));          \
            return 1;                                                                                  \
        }                                                                                              \
    } while (0)

inline int cdiv(int a, int b) { return (a + b - 1) / b; }
inline long round_up(long a, long b) { return (a + b - 1) / b * b; }

// Function attributes (dynamic shared-memory opt-in) are per device: `mask` is a per-call-site bit set of the devices already configured,
// so engines on several devices in one process (nn.DataParallel: one host thread per GPU) each configure their own.
inline bool first_use_on_device(std::atomic<unsigned long long>& mask) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev > 63) return true;
    const unsigned long long bit = 1ull << dev;
    return (mask.fetch_or(bit) & bit) == 0;
}

// Streaming multiprocessors of the current device (132 on an H100 SXM): persistent and grid-stride grids are sized from it.
inline int sm_count() {
    static std::atomic<int> cache[64];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev > 63) dev = 0;
    int n = cache[dev].load();
    if (n == 0) {
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n < 1) n = 132;
        cache[dev].store(n);
    }
    return n;
}

// ---- split-fp16 representation of an fp32 value: x ~= hi + lo, |x - hi - lo| <= 2^-22 |x| + 2^-25
__device__ __forceinline__ void split_f32(float x, __half& hi, __half& lo) {
    hi = __float2half_rn(x);
    lo = __float2half_rn(x - __half2float(hi));
}

// ---- GEMM problem description shared by the SIMT and the wgmma back ends --------------------------
// C[M,N] = sum_s A_s[M,K_s] * W_s[N,K_s]^T  (+ bias[N]) (+ row_bias[row / rows_per_group, N]) ; optional ReLU.
// Each K-segment has its own activation and weight views so concatenated LSTM inputs are never materialised
// (the reference builds torch.cat([prev_h, fc_feats, xt]) every step, AttModel.py:626).
constexpr int kMaxSeg = 3;
struct GemmSeg {
    const float* A = nullptr;      // fp32 activations [M, K], row pitch lda   (SIMT path)
    long lda = 0;
    const float* W = nullptr;      // fp32 weights [N, K], row pitch ldw       (SIMT path)
    long ldw = 0;
    const __half* A_hi = nullptr;  // split planes of A, pitch lda_h (multiple of 8 elements)   (wgmma path)
    const __half* A_lo = nullptr;
    long lda_h = 0;
    const __half* W_hi = nullptr;  // split planes of W, pitch ldw_h
    const __half* W_lo = nullptr;
    long ldw_h = 0;
    int K = 0;
};
struct GemmEpilogue {
    const float* bias = nullptr;        // [N]
    const float* row_bias = nullptr;    // [M / rows_per_group, N], pitch ld_row_bias
    long ld_row_bias = 0;
    int rows_per_group = 1;
    const float* residual = nullptr;    // optional [M, N] added after the bias (pre-norm residual connections), pitch ld_res
    long ld_res = 0;
    int relu = 0;
    float* C = nullptr;                 // fp32 result, pitch ldc (may be null when only the split planes are wanted)
    long ldc = 0;
    __half* C_hi = nullptr;             // optional split planes of the result, pitch ldcs
    __half* C_lo = nullptr;
    long ldcs = 0;
    // Fused nn.LSTMCell epilogue (tensor-core path only).  N = 4H and the weight rows / bias / row-bias / gather-bias columns are
    // gate-interleaved (column 4*j+g holds gate g in (i,f,g,o) of hidden unit j), so one epilogue thread owns all four gates
    // of a unit: c' = sig(f)*c + sig(i)*tanh(g), h' = sig(o)*tanh(c').  C / C_hi / C_lo are unused in this mode.
    int lstm = 0;
    int H = 0;
    const float* c_prev = nullptr;      // [*, H] pitch ld_cprev, read at row src_row[r] (nullptr src_row = identity, < 0 = zero state)
    long ld_cprev = 0;
    const int* src_row = nullptr;
    float* c_out = nullptr;             // [M, H] pitch ld_cout
    long ld_cout = 0;
    const float* gather_bias = nullptr; // optional per-row gathered gate bias: gather_bias[gather_idx[r], 4H] (per-token table)
    long ld_gb = 0;
    const int* gather_idx = nullptr;
    float* h_f = nullptr;               // h' as fp32 and split planes, common pitch ld_h
    __half* h_hi = nullptr;
    __half* h_lo = nullptr;
    long ld_h = 0;
    unsigned long long* trace = nullptr;    // optional phase time stamps of the wgmma kernel ([CTAs][16] %globaltimer values), tools/gemm_trace.py
};

// SFU-based transcendental forms (ex2.approx + fast reciprocal): absolute error < 3e-7 on outputs in [-1, 1].
__device__ __forceinline__ float fast_sigmoid(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }
__device__ __forceinline__ float fast_tanh(float x) {
    const float e = __expf(2.0f * x);
    return 1.0f - __fdividef(2.0f, 1.0f + e);
}
// Four tanh values with four ex2 and ONE reciprocal: 1/y_i is recovered from 1/(y0*y1*y2*y3) by multiplications, which moves work
// from the 16-lane SFU to the FMA pipe (the attention score kernel is SFU-bound).  Arguments are clamped at 10 (tanh(10) rounds to 1
// in fp32), so every y = 1 + e^(2x) stays below 4.9e8 and the product of four below 5.5e34.
__device__ __forceinline__ void fast_tanh4(const float (&x)[4], float (&t)[4]) {
    float y[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) y[i] = 1.0f + __expf(fminf(2.0f * x[i], 20.0f));
    const float p01 = y[0] * y[1], p23 = y[2] * y[3];
    const float r = __fdividef(1.0f, p01 * p23);
    const float r01 = r * p23, r23 = r * p01;
    t[0] = fmaf(-2.0f, r01 * y[1], 1.0f);
    t[1] = fmaf(-2.0f, r01 * y[0], 1.0f);
    t[2] = fmaf(-2.0f, r23 * y[3], 1.0f);
    t[3] = fmaf(-2.0f, r23 * y[2], 1.0f);
}
struct GemmProblem {
    int M = 0, N = 0, nseg = 0;
    GemmSeg seg[kMaxSeg];
    GemmEpilogue epi;
};

enum NumericMode : int {
    kModeSimtFp32 = 0,   // plain fp32 FFMA on CUDA cores (exact reference arithmetic up to summation order)
    kModeTcF16x3 = 1,    // wgmma f16, split-fp16 operands, 3 MMA passes (hi*hi + hi*lo + lo*hi), fp32 accumulate
    kModeTcF16x1 = 2,    // wgmma f16, hi plane only (throughput mode; NOT parity grade)
};

int gemm_simt_launch(const GemmProblem& p, cudaStream_t stream);

// wgmma path: a plan owns the encoded TMA tensor maps; build once per buffer set, launch many times.
struct GemmTcPlan;
GemmTcPlan* gemm_tc_plan_create(const GemmProblem& p, int passes);   // nullptr on failure (see last_error)
int gemm_tc_tile_n(int M, int N);                                     // output-tile width the plan picks for an M x N problem
int gemm_tc_tile_m(int M, int N, int bn);                             // output-tile height of an M-row launch of a plan of width bn
void gemm_tc_plan_destroy(GemmTcPlan* plan);
// Launch-time overrides: the whole epilogue (output pointers, biases, fused-LSTM state pointers change per decode step) and
// M (rows actually valid, <= planned rows; 0 keeps).  The tensor maps keep the planned extents; rows beyond M are computed
// but never stored.
int gemm_tc_plan_launch(GemmTcPlan* plan, const GemmEpilogue* epi_override, int M_override, cudaStream_t stream);
bool gemm_tc_supported(const GemmProblem& p, std::string* why);

int split_planes_launch(const float* x, long ldx, int rows, int cols, __half* hi, __half* lo, long ldh, cudaStream_t stream);
// fp16-range guard of the split conversions (gemm_simt.cu): device-visible flag pointer, host read (optionally clearing it)
int* range_flag_ptr();
int range_flag_read(int reset);
#define CAPB_CHECK_RANGE()                                                                                              \
    do {                                                                                                                \
        if (capb200::range_flag_read(0)) {                                                                              \
            capb200::set_error("a value with |x| >= 65504 (or inf/nan) reached a split-fp16 conversion in an earlier call: results of the "   \
                               "tensor-core modes are invalid for such inputs/weights (DESIGN.md section 3); capb200_range_status(1) clears the flag"); \
            return 1;                                                                                                   \
        }                                                                                                               \
    } while (0)
// gate-interleaving variant for LSTM weights [4H, cols]: destination row 4*j+g <- source row g*H + j
int split_planes_interleave_launch(const float* x, long ldx, int H, int cols, __half* hi, __half* lo, long ldh, cudaStream_t stream);

}  // namespace capb200
