// wgmma GEMM for the caption-decode path:  C[M,N] = sum_s A_s * W_s^T (+bias, +per-group row bias, ReLU)
//
// Replaces the cuBLAS SGEMMs behind nn.Linear / nn.LSTMCell on the hot path (reference call sites:
// captioning/models/AttModel.py:119 att_embed, :172 logit, :628/:635 LSTMCell, :733 h2att).
//
// Numerics.  The reference computes in fp32; parity demands log-probs within 1e-4 and bit-exact greedy ids, which
// single-pass fp16/bf16/tf32 tensor-core products do not deliver.  Operands are therefore kept in HBM as two fp16
// planes (hi = fp16(x), lo = fp16(x - hi): same bytes as fp32) and every K-block issues three f16 wgmmas into
// one fp32 register accumulator:  hi*lo + lo*hi + hi*hi  (the lo*lo term, <= 2^-22 relative, is dropped).
// PASSES == 1 is the throughput mode (hi plane only) and is never used for parity claims.
//
// Structure (persistent: one 128 x BN output tile at a time per CTA, BN = 64, 128 or 160 chosen by the plan, 384 threads = three warpgroups):
//   warpgroup 0     TMA producer (one thread): cp.async.bulk.tensor 2-D boxes [64 k x rows] (128B swizzle) for A_hi, A_lo, W_hi,
//                   W_lo of the current K-block into a STAGES-deep shared-memory ring, mbarrier complete_tx signalling.  It runs ahead
//                   into the next tile while the consumers are in their epilogue.
//   warpgroups 1,2  consumers: each owns 64 rows of the tile, issues wgmma.m64nBNk16 straight from shared-memory descriptors, releases
//                   the ring slot once its wgmmas retired, and runs the fused epilogue (bias / row-bias / ReLU, fp32 store, optional
//                   split-fp16 copy for the next GEMM, or the fused LSTM cell) from the register accumulator.  The epilogue kind is a
//                   template parameter (EpiKind), so each kernel carries the code of one kind only.
// K-segments (up to 3 activation/weight pairs) are walked back to back so concatenated LSTM inputs are never built.
#include <cstdlib>

#include "common.cuh"
#include "ptx.cuh"

namespace capb200 {

namespace {

constexpr int BM = 128;
constexpr int BK = 64;   // fp16 elements: one 128-byte swizzle row
constexpr int kConsumers = 2;                  // consumer warpgroups, 64 accumulator rows each
constexpr int kThreads = 128 * (1 + kConsumers);

struct TcParams {
    CUtensorMap a_hi[kMaxSeg];
    CUtensorMap a_lo[kMaxSeg];
    CUtensorMap w_hi[kMaxSeg];
    CUtensorMap w_lo[kMaxSeg];
    int kblocks[kMaxSeg];
    int nseg;
    int M, N;
    float* C;
    long ldc;
    __half* C_hi;
    __half* C_lo;
    long ldcs;
    const float* bias;
    const float* row_bias;
    long ld_row_bias;
    int rows_per_group;
    int relu;
    const float* residual;
    long ld_res;
    int tiles_m, tiles_n;
    // fused LSTM epilogue (see GemmEpilogue)
    int lstm, H;
    const float* c_prev;
    long ld_cprev;
    const int* src_row;
    float* c_out;
    long ld_cout;
    const float* gather_bias;
    long ld_gb;
    const int* gather_idx;
    float* h_f;
    __half* h_hi;
    __half* h_lo;
    long ld_h;
    unsigned long long* trace;  // optional [CTAs][16] %globaltimer stamps of the kernel's phases (tools/gemm_trace.py); nullptr = off
};

__device__ __forceinline__ unsigned long long gtimer() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
// compiled in only for the TRACE = true instantiation (tools/gemm_trace.py): the production kernels carry no trace branches
#define CAPB_TRACE(slot) do { if (TRACE && p.trace != nullptr) p.trace[(long)blockIdx.x * 16 + (slot)] = gtimer(); } while (0)

template <int BN, int PASSES>
struct TcCfg {
    static constexpr int kPlanes = (PASSES == 3) ? 2 : 1;
    static constexpr uint32_t kABytes = BM * BK * 2;
    static constexpr uint32_t kWBytes = BN * BK * 2;
    static constexpr uint32_t kStageBytes = kPlanes * (kABytes + kWBytes);
    static constexpr uint32_t kRingBudget = 227 * 1024 - 1024 /*align slack*/ - 256 /*barriers*/;   // per-block shared-memory limit
    static constexpr int kStages = kRingBudget / kStageBytes >= 8 ? 8 : kRingBudget / kStageBytes;
    static constexpr uint32_t kSmemBytes = kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;
    static_assert(BN == 64 || BN == 128 || BN == 160, "wgmma wrappers exist for N = 64, 128 and 160");
    static_assert(kWBytes % 1024 == 0, "operand tiles must keep the 1024-byte swizzle-atom alignment");
    static_assert(kStages >= 2, "need at least a double buffer");
    static_assert(kSmemBytes <= 227 * 1024, "shared memory of one H100 block");
};

template <int BN>
__device__ __forceinline__ void wgmma_f16(float* acc, uint64_t da, uint64_t db, int scale_d) {
    if (BN == 160) ptx::wgmma_f16_n160(acc, da, db, scale_d);
    else if (BN == 128) ptx::wgmma_f16_n128(acc, da, db, scale_d);
    else ptx::wgmma_f16_n64(acc, da, db, scale_d);
}

// Epilogue kinds.  Each is its own kernel instantiation: one epilogue that inlined every variant unrolled to 70-170 KB of machine
// code per kernel, more than an SM's instruction cache holds, and every CTA fetched it from L2 at the same moment (DESIGN §6.1).
enum EpiKind : int {
    kEpiStore = 0,    // fp32 C
    kEpiPlanes = 1,   // optional fp32 C + split fp16 planes C_hi / C_lo
    kEpiLstm = 2,     // fused nn.LSTMCell: c_out, h_f, optional h_hi / h_lo
};

// Accumulator element acc[4j + e] of thread (w, lane) is row r0 + 8 * (e / 2), column c0 + 8j + e % 2, with r0 = m0 + 16w + lane/4 and
// c0 = n0 + 2 * (lane % 4).  Every column pair starts at an even column.
//
// Bias, row bias, gathered bias, residual, then ReLU, each applied to the whole tile in turn: every element gets the same adds in the
// same order as one element at a time would give it, each option is tested once per tile, and all of the tile's loads come before its
// first store.  Elements outside [M, N) are left alone; no kind stores them.
template <int BN>
__device__ __forceinline__ void epi_adds(const TcParams& p, float* acc, int r0, int c0) {
    const int ncol = p.N - c0;                                  // column c0 + k is in range iff k < ncol
    const int lim[2] = {r0 < p.M ? ncol : 0, r0 + 8 < p.M ? ncol : 0};     // ... and on a row in range
    if (p.bias != nullptr) {
        const float* b = p.bias + c0;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                if (8 * j + e < ncol) {
                    const float x = __ldg(b + 8 * j + e);
                    acc[4 * j + e] += x;
                    acc[4 * j + 2 + e] += x;
                }
            }
        }
    }
    // row bias, gathered bias, residual: one row pointer per accumulator row, indexed by column like the bias.  One loop body serves
    // all three (not unrolled: the code is fetched once per tile whichever options are on).
    const float* tab[3][2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int row = lim[h] > 0 ? r0 + 8 * h : 0;
        tab[0][h] = p.row_bias != nullptr ? p.row_bias + (long)(row / p.rows_per_group) * p.ld_row_bias + c0 : nullptr;
        tab[1][h] = p.gather_bias != nullptr ? p.gather_bias + (long)(lim[h] > 0 ? p.gather_idx[row] : 0) * p.ld_gb + c0 : nullptr;
        tab[2][h] = p.residual != nullptr ? p.residual + (long)row * p.ld_res + c0 : nullptr;
    }
#pragma unroll 1
    for (int t = 0; t < 3; ++t) {
        const float* const t0 = t == 0 ? tab[0][0] : t == 1 ? tab[1][0] : tab[2][0];
        const float* const t1 = t == 0 ? tab[0][1] : t == 1 ? tab[1][1] : tab[2][1];
        if (t0 == nullptr) continue;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int k = 8 * j + (e & 1);
                if (k < lim[e >> 1]) acc[4 * j + e] += (e >> 1 ? t1 : t0)[k];
            }
        }
    }
    if (p.relu) {
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = fmaxf(acc[i], 0.0f);
    }
}

// Fused LSTM cell.  Gates (i,f,g,o) of hidden unit c/4 sit in lanes 2k (i,f) and 2k+1 (g,o): the even lane finishes the unit for row r0,
// the odd lane for row r0 + 8, each taking the two gates it lacks from its neighbour.  src_row and the c_prev values of the thread's
// BN/8 units are loaded before the first store.
template <int BN>
__device__ __forceinline__ void epi_lstm(const TcParams& p, const float* acc, int r0, int c0, int lane) {
    const bool odd = lane & 1;
    const int row = r0 + (odd ? 8 : 0);
    const int u0 = c0 >> 2;                                     // unit of column pair j is u0 + 2j
    const bool row_ok = row < p.M;
    int src = row;
    if (p.src_row != nullptr && row_ok) src = p.src_row[row];
    const float* cprev = (src >= 0 && p.c_prev != nullptr) ? p.c_prev + (long)src * p.ld_cprev : nullptr;
    float cp[BN / 8];
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) cp[j] = (row_ok && cprev != nullptr && u0 + 2 * j < p.H) ? cprev[u0 + 2 * j] : 0.0f;
    float* const c_out = p.c_out + (long)row * p.ld_cout;
    float* const h_f = p.h_f + (long)row * p.ld_h;
    __half* const h_hi = p.h_hi + (long)row * p.ld_h;
    __half* const h_lo = p.h_lo + (long)row * p.ld_h;
    const bool planes = p.h_hi != nullptr;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
        const float* v = acc + 4 * j;
        const float s0 = __shfl_xor_sync(0xffffffffu, odd ? v[0] : v[2], 1);
        const float s1 = __shfl_xor_sync(0xffffffffu, odd ? v[1] : v[3], 1);
        const float gi = odd ? s0 : v[0], gf = odd ? s1 : v[1], gg = odd ? v[2] : s0, go = odd ? v[3] : s1;
        const int unit = u0 + 2 * j;
        if (row_ok && unit < p.H) {
            const float cn = fast_sigmoid(gf) * cp[j] + fast_sigmoid(gi) * fast_tanh(gg);
            const float hn = fast_sigmoid(go) * fast_tanh(cn);
            c_out[unit] = cn;
            h_f[unit] = hn;
            if (planes) {
                __half hh, hl;
                split_f32(hn, hh, hl);
                h_hi[unit] = hh;
                h_lo[unit] = hl;
            }
        }
    }
}

// fp32 C and / or the split planes of rows r0, r0 + 8.  Columns come in pairs starting at an even column, so whether the pairs of a row
// can be stored as vectors depends on the row alone: a row whose pointers are aligned and whose columns are all in range takes the
// vector loop, any other the element loop.
template <int BN, bool PLANES>
__device__ __forceinline__ void epi_store(const TcParams& p, const float* acc, int r0, int c0) {
    const int ncol = p.N - c0;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int row = r0 + 8 * h;
        if (row >= p.M) continue;
        if (p.C != nullptr) {
            float* const dst = p.C + (long)row * p.ldc + c0;
            if (ncol >= BN && (reinterpret_cast<uintptr_t>(dst) & 7) == 0) {
#pragma unroll
                for (int j = 0; j < BN / 8; ++j) *reinterpret_cast<float2*>(dst + 8 * j) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
            } else {
#pragma unroll
                for (int j = 0; j < BN / 8; ++j) {
                    if (8 * j < ncol) dst[8 * j] = acc[4 * j + 2 * h];
                    if (8 * j + 1 < ncol) dst[8 * j + 1] = acc[4 * j + 2 * h + 1];
                }
            }
        }
        if (PLANES) {
            __half* const dh = p.C_hi + (long)row * p.ldcs + c0;
            __half* const dl = p.C_lo + (long)row * p.ldcs + c0;
            if (ncol >= BN && ((reinterpret_cast<uintptr_t>(dh) | reinterpret_cast<uintptr_t>(dl)) & 3) == 0) {
#pragma unroll
                for (int j = 0; j < BN / 8; ++j) {
                    __half h0, l0, h1, l1;
                    split_f32(acc[4 * j + 2 * h], h0, l0);
                    split_f32(acc[4 * j + 2 * h + 1], h1, l1);
                    *reinterpret_cast<__half2*>(dh + 8 * j) = __halves2half2(h0, h1);
                    *reinterpret_cast<__half2*>(dl + 8 * j) = __halves2half2(l0, l1);
                }
            } else {
#pragma unroll
                for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        __half hi, lo;
                        split_f32(acc[4 * j + 2 * h + e], hi, lo);
                        if (8 * j + e < ncol) { dh[8 * j + e] = hi; dl[8 * j + e] = lo; }
                    }
                }
            }
        }
    }
}

// Drains this warpgroup's 64 x BN accumulator (layout above).
template <int BN, int EPI>
__device__ __forceinline__ void epilogue_tile(const TcParams& p, float* acc, int m0, int n0, int tid) {
    const int warp = tid >> 5, lane = tid & 31;
    const int r0 = m0 + warp * 16 + (lane >> 2);
    const int c0 = n0 + 2 * (lane & 3);
    epi_adds<BN>(p, acc, r0, c0);
    if (EPI == kEpiLstm) epi_lstm<BN>(p, acc, r0, c0, lane);
    else epi_store<BN, EPI == kEpiPlanes>(p, acc, r0, c0);
}

// Persistent schedule: gridDim.x = min(tiles, SMs); CTA b walks tiles b, b + gridDim.x, ... in m-fastest order so that concurrently
// running CTAs share the same weight columns (the W tile comes from HBM once, then from L2).
template <int BN, int PASSES, int EPI, bool TRACE = false>
__global__ void __launch_bounds__(kThreads, 1) gemm_tc_kernel(const __grid_constant__ TcParams p) {
    using Cfg = TcCfg<BN, PASSES>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::kStages * Cfg::kStageBytes);
    uint64_t* empty_bar = full_bar + Cfg::kStages;

    const int wg = threadIdx.x >> 7;
    const int n_tiles = p.tiles_m * p.tiles_n;

    if (threadIdx.x == 0) {
        for (int s = 0; s < p.nseg; ++s) {
            ptx::prefetch_tmap(&p.a_hi[s]);
            ptx::prefetch_tmap(&p.w_hi[s]);
            if (PASSES == 3) {
                ptx::prefetch_tmap(&p.a_lo[s]);
                ptx::prefetch_tmap(&p.w_lo[s]);
            }
        }
        for (int i = 0; i < Cfg::kStages; ++i) {
            ptx::mbar_init(&full_bar[i], 1);
            ptx::mbar_init(&empty_bar[i], kConsumers);        // one release per consumer warpgroup
        }
        ptx::fence_mbar_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) CAPB_TRACE(0);                       // set-up done

    if (wg == 0) {
        if (threadIdx.x == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
                const int m0 = (t % p.tiles_m) * BM;
                const int n0 = (t / p.tiles_m) * BN;
                for (int s = 0; s < p.nseg; ++s) {
                    for (int kb = 0; kb < p.kblocks[s]; ++kb) {
                        ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
                        uint8_t* st = smem + stage * Cfg::kStageBytes;
                        uint8_t* a_hi = st;
                        uint8_t* a_lo = st + Cfg::kABytes;
                        uint8_t* w_hi = st + Cfg::kABytes * Cfg::kPlanes;
                        uint8_t* w_lo = st + Cfg::kABytes * 2 + Cfg::kWBytes;
                        ptx::mbar_arrive_expect_tx(&full_bar[stage], Cfg::kStageBytes);
                        ptx::tma_load_2d(a_hi, &p.a_hi[s], &full_bar[stage], kb * BK, m0);
                        ptx::tma_load_2d(w_hi, &p.w_hi[s], &full_bar[stage], kb * BK, n0);
                        if (PASSES == 3) {
                            ptx::tma_load_2d(a_lo, &p.a_lo[s], &full_bar[stage], kb * BK, m0);
                            ptx::tma_load_2d(w_lo, &p.w_lo[s], &full_bar[stage], kb * BK, n0);
                        }
                        if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
                    }
                }
            }
        }
    } else {
        const int cw = wg - 1;                                  // rows [64 cw, 64 cw + 64) of every tile
        const int tid = threadIdx.x & 127;
        const uint32_t a_off = cw * 64 * 128;                   // 64 rows of 128 bytes: a whole number of swizzle atoms
        int stage = 0;
        uint32_t phase = 0;
        int it = 0;
        for (int t = blockIdx.x; t < n_tiles; t += gridDim.x, ++it) {
            const int m0 = (t % p.tiles_m) * BM;
            const int n0 = (t / p.tiles_m) * BN;
            float acc[BN / 2];
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) acc[i] = 0.0f;
            for (int s = 0; s < p.nseg; ++s) {
                for (int kb = 0; kb < p.kblocks[s]; ++kb) {
                    ptx::mbar_wait(&full_bar[stage], phase);
                    if (TRACE && it == 0 && s == 0 && kb == 0 && tid == 0 && cw == 0) CAPB_TRACE(1);    // first operands landed
                    const uint32_t st = ptx::smem_u32(smem + stage * Cfg::kStageBytes);
                    const uint32_t a_hi = st + a_off;
                    const uint32_t a_lo = st + Cfg::kABytes + a_off;                  // only valid when PASSES == 3
                    const uint32_t w_hi = st + Cfg::kABytes * Cfg::kPlanes;
                    const uint32_t w_lo = st + Cfg::kABytes * 2 + Cfg::kWBytes;       // only valid when PASSES == 3
#pragma unroll
                    for (int i = 0; i < BN / 2; ++i) ptx::reg_fence(acc[i]);
                    ptx::wgmma_fence();
#pragma unroll
                    for (int k = 0; k < BK / 16; ++k) {
                        const uint32_t koff = k * 32;   // 16 fp16 = 32 bytes inside the 128-byte swizzle row
                        if (PASSES == 3) {
                            wgmma_f16<BN>(acc, ptx::make_smem_desc_sw128(a_hi + koff), ptx::make_smem_desc_sw128(w_lo + koff), 1);
                            wgmma_f16<BN>(acc, ptx::make_smem_desc_sw128(a_lo + koff), ptx::make_smem_desc_sw128(w_hi + koff), 1);
                        }
                        wgmma_f16<BN>(acc, ptx::make_smem_desc_sw128(a_hi + koff), ptx::make_smem_desc_sw128(w_hi + koff), 1);
                    }
                    ptx::wgmma_commit();
                    ptx::wgmma_wait<0>();
#pragma unroll
                    for (int i = 0; i < BN / 2; ++i) ptx::reg_fence(acc[i]);
                    if (tid == 0) ptx::mbar_arrive(&empty_bar[stage]);                // this warpgroup no longer reads the slot
                    if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
                }
            }
            if (TRACE && it < 2 && tid == 0 && cw == 0) CAPB_TRACE(2 + it);          // main loop of tile `it` done
            epilogue_tile<BN, EPI>(p, acc, m0 + cw * 64, n0, tid);
            if (TRACE && it < 2 && tid == 0 && cw == 0) CAPB_TRACE(6 + it);          // epilogue of tile `it` done
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) CAPB_TRACE(8);                       // every role is done
}

// ---- host side ------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (fn == nullptr) {
        void* sym = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres) != cudaSuccess || sym == nullptr) {
            return nullptr;
        }
        fn = reinterpret_cast<EncodeTiledFn>(sym);
    }
    return fn;
}

// fp16 plane [rows, K] with row pitch `pitch` elements; box = 64 (K) x box_rows, 128-byte swizzle, zero OOB fill.
bool encode_plane(CUtensorMap* map, const __half* base, long rows, long K, long pitch, int box_rows, std::string* err) {
    EncodeTiledFn fn = get_encode_fn();
    if (fn == nullptr) { *err = "cuTensorMapEncodeTiled entry point not available"; return false; }
    cuuint64_t gdim[2] = {static_cast<cuuint64_t>(K), static_cast<cuuint64_t>(rows)};
    cuuint64_t gstride[1] = {static_cast<cuuint64_t>(pitch) * 2};
    cuuint32_t box[2] = {static_cast<cuuint32_t>(BK), static_cast<cuuint32_t>(box_rows)};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(base), gdim, gstride, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { *err = "cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r); return false; }
    return true;
}

template <int BN, int PASSES, int EPI, bool TRACE = false>
int launch_cfg(const TcParams& prm, cudaStream_t stream) {
    using Cfg = TcCfg<BN, PASSES>;
    static std::atomic<unsigned long long> attr_set{0};
    if (first_use_on_device(attr_set)) {
        CAPB_CHECK_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<BN, PASSES, EPI, TRACE>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
    }
    TcParams prm2 = prm;
    prm2.tiles_n = cdiv(prm.N, BN);
    prm2.tiles_m = cdiv(prm.M, BM);
    const int n_tiles = prm2.tiles_n * prm2.tiles_m;
    const int sms = sm_count();
    gemm_tc_kernel<BN, PASSES, EPI, TRACE><<<n_tiles < sms ? n_tiles : sms, kThreads, Cfg::kSmemBytes, stream>>>(prm2);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// kind x BN x passes, plus the traced 3-pass kernels (capb200_decode_gemm with a trace buffer)
template <int EPI>
int launch_kind(int bn, int passes, const TcParams& prm, cudaStream_t stream) {
    if (prm.trace != nullptr) {
        if (bn == 160) return launch_cfg<160, 3, EPI, true>(prm, stream);
        return bn == 128 ? launch_cfg<128, 3, EPI, true>(prm, stream) : launch_cfg<64, 3, EPI, true>(prm, stream);
    }
    if (bn == 160) return passes == 3 ? launch_cfg<160, 3, EPI>(prm, stream) : launch_cfg<160, 1, EPI>(prm, stream);
    if (bn == 128) return passes == 3 ? launch_cfg<128, 3, EPI>(prm, stream) : launch_cfg<128, 1, EPI>(prm, stream);
    return passes == 3 ? launch_cfg<64, 3, EPI>(prm, stream) : launch_cfg<64, 1, EPI>(prm, stream);
}

}  // namespace

struct GemmTcPlan {
    TcParams prm;
    int passes;
    int bn;
};

static void fill_epilogue(TcParams& t, const GemmEpilogue& e) {
    t.C = e.C; t.ldc = e.ldc;
    t.C_hi = e.C_hi; t.C_lo = e.C_lo; t.ldcs = e.ldcs;
    t.bias = e.bias; t.row_bias = e.row_bias; t.ld_row_bias = e.ld_row_bias;
    t.rows_per_group = e.rows_per_group < 1 ? 1 : e.rows_per_group;
    t.relu = e.relu;
    t.residual = e.residual; t.ld_res = e.ld_res;
    t.lstm = e.lstm; t.H = e.H;
    t.c_prev = e.c_prev; t.ld_cprev = e.ld_cprev; t.src_row = e.src_row;
    t.c_out = e.c_out; t.ld_cout = e.ld_cout;
    t.gather_bias = e.gather_bias; t.ld_gb = e.ld_gb; t.gather_idx = e.gather_idx;
    t.h_f = e.h_f; t.h_hi = e.h_hi; t.h_lo = e.h_lo; t.ld_h = e.ld_h;
    t.trace = e.trace;
}

bool gemm_tc_supported(const GemmProblem& p, std::string* why) {
    auto bad = [&](const char* m) { if (why) *why = m; return false; };
    if (p.nseg < 1 || p.nseg > kMaxSeg) return bad("1..3 K-segments");
    for (int s = 0; s < p.nseg; ++s) {
        const GemmSeg& g = p.seg[s];
        if (g.A_hi == nullptr || g.W_hi == nullptr) return bad("split planes missing");
        if ((g.lda_h & 7) || (g.ldw_h & 7)) return bad("plane pitch must be a multiple of 8 elements (16 bytes)");
        if ((reinterpret_cast<uintptr_t>(g.A_hi) & 15) || (reinterpret_cast<uintptr_t>(g.W_hi) & 15)) return bad("plane base must be 16-byte aligned");
        if (g.K < 1) return bad("empty K-segment");
    }
    return true;
}

// Tile width.  Problems with fewer 128-wide tiles than half the SMs are latency-bound: 64-wide tiles double the CTAs.  Otherwise the
// width of 128 or 160 with the fewest waves x BN; 160 pays for the 1280 x 4000 LSTM gates (2 waves instead of 3 on 132 SMs, measured on
// an H100 80GB HBM3 with tools/decode_gemm_rate.py).  Ties go to 128, the narrower tile that wastes fewer columns on a ragged last n-tile;
// no measurement has yet compared the two widths at a tie.
int gemm_tc_tile_n(int M, int N) {
    const int sms = sm_count();
    const int tiles_m = cdiv(M, BM);
    if (tiles_m * cdiv(N, 128) < sms / 2 && N > 64) return 64;
    const long cost128 = (long)cdiv(tiles_m * cdiv(N, 128), sms) * 128;
    const long cost160 = (long)cdiv(tiles_m * cdiv(N, 160), sms) * 160;
    return cost160 < cost128 ? 160 : 128;
}

GemmTcPlan* gemm_tc_plan_create(const GemmProblem& p, int passes) {
    std::string why;
    if (!gemm_tc_supported(p, &why)) { set_error("gemm_tc: unsupported problem: " + why); return nullptr; }
    if (passes != 1 && passes != 3) { set_error("gemm_tc: passes must be 1 or 3"); return nullptr; }
    GemmTcPlan* plan = new GemmTcPlan();
    memset(&plan->prm, 0, sizeof(TcParams));
    plan->passes = passes;
    plan->bn = gemm_tc_tile_n(p.M, p.N);
    TcParams& t = plan->prm;
    t.nseg = p.nseg;
    t.M = p.M;
    t.N = p.N;
    std::string err;
    for (int s = 0; s < p.nseg; ++s) {
        const GemmSeg& g = p.seg[s];
        t.kblocks[s] = cdiv(g.K, BK);
        bool ok = encode_plane(&t.a_hi[s], g.A_hi, p.M, g.K, g.lda_h, BM, &err) &&
                  encode_plane(&t.w_hi[s], g.W_hi, p.N, g.K, g.ldw_h, plan->bn, &err);
        if (ok && passes == 3) {
            if (g.A_lo == nullptr || g.W_lo == nullptr) { err = "lo planes missing for 3-pass mode"; ok = false; }
            ok = ok && encode_plane(&t.a_lo[s], g.A_lo, p.M, g.K, g.lda_h, BM, &err) &&
                 encode_plane(&t.w_lo[s], g.W_lo, p.N, g.K, g.ldw_h, plan->bn, &err);
        }
        if (!ok) { set_error("gemm_tc: " + err); delete plan; return nullptr; }
    }
    fill_epilogue(t, p.epi);
    return plan;
}

void gemm_tc_plan_destroy(GemmTcPlan* plan) { delete plan; }

int gemm_tc_plan_launch(GemmTcPlan* plan, const GemmEpilogue* epi_override, int M_override, cudaStream_t stream) {
    TcParams prm = plan->prm;
    if (epi_override != nullptr) fill_epilogue(prm, *epi_override);
    if (M_override > 0) {
        if (M_override > prm.M) { set_error("gemm_tc: M override exceeds the planned row count"); return 1; }
        prm.M = M_override;
    }
    if (prm.lstm && (prm.N != 4 * prm.H || prm.c_out == nullptr || prm.h_f == nullptr)) {
        set_error("gemm_tc: fused LSTM epilogue needs N == 4H, c_out and h_f");
        return 1;
    }
    if (prm.M <= 0 || prm.N <= 0) return 0;
    // the kind follows the epilogue this launch asks for: launches override the planned one whole
    const int kind = prm.lstm ? kEpiLstm : prm.C_hi != nullptr ? kEpiPlanes : kEpiStore;
    if (prm.trace != nullptr && plan->passes != 3) { set_error("gemm_tc: the traced kernel is the 3-pass one"); return 1; }
    if (kind == kEpiLstm) return launch_kind<kEpiLstm>(plan->bn, plan->passes, prm, stream);
    if (kind == kEpiPlanes) return launch_kind<kEpiPlanes>(plan->bn, plan->passes, prm, stream);
    return launch_kind<kEpiStore>(plan->bn, plan->passes, prm, stream);
}

}  // namespace capb200
