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
//                   into the next tile.  40 registers (setmaxnreg), the consumers 232.
//   warpgroups 1,2  ping-pong consumers: warpgroup 1 runs the CTA's even tiles, warpgroup 2 its odd ones, each holding the whole
//                   128 x BN accumulator as two m64 halves.  They take turns at the main loop (wgmma.m64nBNk16 straight from
//                   shared-memory descriptors, the ring slot released once the wgmmas retired), so one tile's fused epilogue (bias /
//                   row-bias / ReLU, fp32 store, optional split-fp16 copy for the next GEMM, or the fused LSTM cell) runs from registers
//                   under the next tile's main loop; only a CTA's last epilogue is exposed.  The epilogue kind is a template parameter
//                   (EpiKind), so each kernel carries the code of one kind only.
// gemm_tc256_kernel is the cooperative schedule of the same roles over 256 x BN tiles (BN 128 or 160): both consumer warpgroups read
// every stage, each its own 128 rows of A against the one W tile, so a K-block feeds twice the outputs for 1.4-1.5x the bytes.  At
// three passes two stages fit.  gemm_tc_tile_m picks the schedule per launch.
// On an H100 80GB HBM3 at a 400 W power limit, the ping-pong schedule and the vectorised LSTM stores take the UpDown decode step's LSTM
// gate GEMMs from 3.34 to 3.02-3.06 ms (att_lstm) and 4.10-4.14 to 3.74-3.81 ms (lang_lstm) per batch; logit and h2att are unchanged
// (DESIGN §5.1).
// K-segments (up to 3 activation/weight pairs) are walked back to back so concatenated LSTM inputs are never built.
#include <cstdlib>
#include <cstring>

#include "common.cuh"
#include "ptx.cuh"

namespace capb200 {

namespace {

constexpr int BM = 128;
constexpr int BK = 64;   // fp16 elements: one 128-byte swizzle row
constexpr int kConsumers = 2;                  // consumer warpgroups, one whole tile each, taking turns
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

// TM: rows of A per stage, BM for the ping-pong kernel and 2 * BM for the cooperative one (gemm_tc256_kernel)
template <int BN, int PASSES, int TM = BM>
struct TcCfg {
    static constexpr int kTileM = TM;
    static constexpr int kPasses = PASSES;
    static constexpr int kPlanes = (PASSES == 3) ? 2 : 1;
    static constexpr uint32_t kABytes = TM * BK * 2;
    static constexpr uint32_t kWBytes = BN * BK * 2;
    static constexpr uint32_t kStageBytes = kPlanes * (kABytes + kWBytes);
    static constexpr uint32_t kRingBudget = 227 * 1024 - 1024 /*align slack*/ - 256 /*barriers*/;   // per-block shared-memory limit
    static constexpr int kStages = kRingBudget / kStageBytes >= 8 ? 8 : kRingBudget / kStageBytes;
    static constexpr uint32_t kSmemBytes = kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;
    static_assert(BN == 64 || BN == 128 || BN == 160, "wgmma wrappers exist for N = 64, 128 and 160");
    static_assert(TM == BM || TM == 2 * BM, "one or two 128-row A boxes per plane");
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

// Fused LSTM cell.  Gates (i,f,g,o) of hidden unit c/4 sit in lanes 2k (i,f) and 2k+1 (g,o) of a quad: the even lane takes the unit for
// row r0, the odd lane for row r0 + 8, each taking the two gates it lacks from its neighbour (shfl.xor 1).  Quad lanes q and q ^ 2 then
// hold the even and the odd units of the same row; they trade (shfl.xor 2) so that each lane holds runs of 4 consecutive units of its
// row, one run per 16 gate columns, and c_prev, c_out and h_f move as 16-byte vectors, h_hi and h_lo as 8-byte ones.  A row whose
// pointers are not aligned for that, or whose units run past H, takes the element path.  Units of run k of lane q: u0 + 8k + 4 * (q >> 1)
// + o, o = 0..3; unit o of run k comes from column pair j = 4k + (o >> 1) + 2 * (o & 1).  Every load comes before the first store.
// TRACE: thread `slot >= 0` stamps slots slot, slot + 1, slot + 2 when its c_prev values have landed, the cell math is done and its
// last store is issued.
template <int BN, bool TRACE>
__device__ __forceinline__ void epi_lstm(const TcParams& p, float* acc, int r0, int c0, int lane, int slot) {
    constexpr int kRuns = BN / 32;
    const bool odd = lane & 1;
    const bool upper = lane & 2;
    const int row = r0 + (odd ? 8 : 0);
    const int u0 = ((c0 - 2 * (lane & 3)) >> 2) + (upper ? 4 : 0);   // first unit of run 0
    const bool row_ok = row < p.M;
    const bool full = u0 + 8 * (kRuns - 1) + 4 <= p.H;                  // every unit of the lane in range
    int src = row;
    if (p.src_row != nullptr && row_ok) src = p.src_row[row];
    const float* cprev = (row_ok && src >= 0 && p.c_prev != nullptr) ? p.c_prev + (long)src * p.ld_cprev + u0 : nullptr;
    float cp[BN / 8];
    if (cprev != nullptr && full && (reinterpret_cast<uintptr_t>(cprev) & 15) == 0) {
#pragma unroll
        for (int k = 0; k < kRuns; ++k) {
            const float4 v = *reinterpret_cast<const float4*>(cprev + 8 * k);
            cp[4 * k] = v.x; cp[4 * k + 1] = v.y; cp[4 * k + 2] = v.z; cp[4 * k + 3] = v.w;
        }
    } else {
#pragma unroll
        for (int i = 0; i < BN / 8; ++i) {
            const int du = 8 * (i / 4) + i % 4;
            cp[i] = (cprev != nullptr && u0 + du < p.H) ? cprev[du] : 0.0f;
        }
    }
    if (TRACE && slot >= 0) {
        float s = 0.0f;
#pragma unroll
        for (int i = 0; i < BN / 8; ++i) s += cp[i];
        asm volatile("" ::"f"(s));
        CAPB_TRACE(slot);
    }
    __syncwarp();                                               // the load paths above diverge; the shuffles below need no fallback
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {                          // gates of unit (u0 - 4 * upper) + 2j + (upper): acc[4j .. 4j + 3] = i, f, g, o
        float* v = acc + 4 * j;
        const float s0 = __shfl_xor_sync(0xffffffffu, odd ? v[0] : v[2], 1);
        const float s1 = __shfl_xor_sync(0xffffffffu, odd ? v[1] : v[3], 1);
        const float gi = odd ? s0 : v[0], gf = odd ? s1 : v[1], gg = odd ? v[2] : s0, go = odd ? v[3] : s1;
        v[0] = gi; v[1] = gf; v[2] = gg; v[3] = go;
    }
#pragma unroll
    for (int k = 0; k < kRuns; ++k) {                           // lower lane keeps pairs 4k, 4k + 1, upper lane pairs 4k + 2, 4k + 3
#pragma unroll
        for (int t = 0; t < 2; ++t) {
            float* x = acc + 4 * (4 * k + t);                   // becomes unit o = 2t of run k
            float* y = acc + 4 * (4 * k + 2 + t);               // becomes unit o = 2t + 1
#pragma unroll
            for (int g = 0; g < 4; ++g) {
                const float keep = upper ? y[g] : x[g];
                const float recv = __shfl_xor_sync(0xffffffffu, upper ? x[g] : y[g], 2);
                x[g] = upper ? recv : keep;
                y[g] = upper ? keep : recv;
            }
        }
    }
    float cn[BN / 8], hn[BN / 8];
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
        const int k = i / 4, o = i % 4;
        const float* g = acc + 4 * (4 * k + (o >> 1) + 2 * (o & 1));
        cn[i] = fast_sigmoid(g[1]) * cp[i] + fast_sigmoid(g[0]) * fast_tanh(g[2]);
        hn[i] = fast_sigmoid(g[3]) * fast_tanh(cn[i]);
    }
    if (TRACE && slot >= 0) {
        float s = 0.0f;
#pragma unroll
        for (int i = 0; i < BN / 8; ++i) s += hn[i];
        asm volatile("" ::"f"(s));
        CAPB_TRACE(slot + 1);
    }
    if (row_ok) {
        float* const c_out = p.c_out + (long)row * p.ld_cout + u0;
        float* const h_f = p.h_f + (long)row * p.ld_h + u0;
        __half* const h_hi = p.h_hi + (long)row * p.ld_h + u0;
        __half* const h_lo = p.h_lo + (long)row * p.ld_h + u0;
        const bool planes = p.h_hi != nullptr;
        const uintptr_t a16 = reinterpret_cast<uintptr_t>(c_out) | reinterpret_cast<uintptr_t>(h_f);
        const uintptr_t a8 = planes ? reinterpret_cast<uintptr_t>(h_hi) | reinterpret_cast<uintptr_t>(h_lo) : 0;
        if (full && (a16 & 15) == 0 && (a8 & 7) == 0) {
#pragma unroll
            for (int k = 0; k < kRuns; ++k) {
                const float* c = cn + 4 * k;
                const float* h = hn + 4 * k;
                *reinterpret_cast<float4*>(c_out + 8 * k) = make_float4(c[0], c[1], c[2], c[3]);
                *reinterpret_cast<float4*>(h_f + 8 * k) = make_float4(h[0], h[1], h[2], h[3]);
                if (planes) {
                    __half hh[4], hl[4];
#pragma unroll
                    for (int o = 0; o < 4; ++o) split_f32(h[o], hh[o], hl[o]);
                    const __half2 hi01 = __halves2half2(hh[0], hh[1]), hi23 = __halves2half2(hh[2], hh[3]);
                    const __half2 lo01 = __halves2half2(hl[0], hl[1]), lo23 = __halves2half2(hl[2], hl[3]);
                    *reinterpret_cast<uint2*>(h_hi + 8 * k) = make_uint2(*reinterpret_cast<const uint32_t*>(&hi01), *reinterpret_cast<const uint32_t*>(&hi23));
                    *reinterpret_cast<uint2*>(h_lo + 8 * k) = make_uint2(*reinterpret_cast<const uint32_t*>(&lo01), *reinterpret_cast<const uint32_t*>(&lo23));
                }
            }
        } else {
#pragma unroll
            for (int i = 0; i < BN / 8; ++i) {
                const int du = 8 * (i / 4) + i % 4;
                if (u0 + du < p.H) {
                    c_out[du] = cn[i];
                    h_f[du] = hn[i];
                    if (planes) {
                        __half hh, hl;
                        split_f32(hn[i], hh, hl);
                        h_hi[du] = hh;
                        h_lo[du] = hl;
                    }
                }
            }
        }
    }
    if (TRACE && slot >= 0) CAPB_TRACE(slot + 2);
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

// Drains 64 rows x BN of a warpgroup's accumulator (layout above).  TRACE: `slot` as for epi_lstm.
template <int BN, int EPI, bool TRACE>
__device__ __forceinline__ void epilogue_tile(const TcParams& p, float* acc, int m0, int n0, int tid, int slot) {
    const int warp = tid >> 5, lane = tid & 31;
    const int r0 = m0 + warp * 16 + (lane >> 2);
    const int c0 = n0 + 2 * (lane & 3);
    epi_adds<BN>(p, acc, r0, c0);
    if (EPI == kEpiLstm) epi_lstm<BN, TRACE>(p, acc, r0, c0, lane, slot);
    else epi_store<BN, EPI == kEpiPlanes>(p, acc, r0, c0);
}

// Drains a warpgroup's 128 rows: rows 0..63 from acc0, then rows 64..127 moved into acc0, so the epilogue's code exists once, indexed
// statically.  `slot` stamps the first 64 rows only.
template <int BN, int EPI, bool TRACE>
__device__ __forceinline__ void epilogue_rows128(const TcParams& p, float* acc0, const float* acc1, int m0, int n0, int tid, int slot) {
#pragma unroll 1
    for (int h = 0; h < 2; ++h) {
        epilogue_tile<BN, EPI, TRACE>(p, acc0, m0 + 64 * h, n0, tid, h == 0 ? slot : -1);
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc0[i] = acc1[i];
    }
}

// Set-up shared by both schedules (thread 0): the tensor maps prefetched, the ring's barriers initialised.  A stage's empty barrier
// takes one arrival per warpgroup that reads the stage.
template <int PASSES>
__device__ __forceinline__ void init_ring(const TcParams& p, uint64_t* full_bar, uint64_t* empty_bar, int stages, int readers) {
    for (int s = 0; s < p.nseg; ++s) {
        ptx::prefetch_tmap(&p.a_hi[s]);
        ptx::prefetch_tmap(&p.w_hi[s]);
        if (PASSES == 3) {
            ptx::prefetch_tmap(&p.a_lo[s]);
            ptx::prefetch_tmap(&p.w_lo[s]);
        }
    }
    for (int i = 0; i < stages; ++i) {
        ptx::mbar_init(&full_bar[i], 1);
        ptx::mbar_init(&empty_bar[i], readers);
    }
}

// Producer: K-block kb of segment s into one stage, laid out [A_hi | A_lo | W_hi | W_lo] (the lo planes only for three passes).  A's
// kTileM rows from m0 come as 128-row boxes (the plan's A maps serve both schedules), W's BN rows from n0 as one box.
template <typename Cfg>
__device__ __forceinline__ void fill_stage(const TcParams& p, uint8_t* st, uint64_t* bar, int s, int kb, int m0, int n0) {
    uint8_t* a_hi = st;
    uint8_t* a_lo = st + Cfg::kABytes;
    uint8_t* w_hi = st + Cfg::kABytes * Cfg::kPlanes;
    uint8_t* w_lo = w_hi + Cfg::kWBytes;
    ptx::mbar_arrive_expect_tx(bar, Cfg::kStageBytes);
#pragma unroll
    for (int r = 0; r < Cfg::kTileM; r += BM) ptx::tma_load_2d(a_hi + r * BK * 2, &p.a_hi[s], bar, kb * BK, m0 + r);
    ptx::tma_load_2d(w_hi, &p.w_hi[s], bar, kb * BK, n0);
    if (Cfg::kPasses == 3) {
#pragma unroll
        for (int r = 0; r < Cfg::kTileM; r += BM) ptx::tma_load_2d(a_lo + r * BK * 2, &p.a_lo[s], bar, kb * BK, m0 + r);
        ptx::tma_load_2d(w_lo, &p.w_lo[s], bar, kb * BK, n0);
    }
}

// Consumer: one K-block of a warpgroup's 128 rows (two m64 halves of A at a_hi / a_lo, 128-byte swizzled rows) against the stage's W,
// issued and retired.  Per k16 slice the same hi*lo, lo*hi, hi*hi order into each half (per element the sums of a 64-row warpgroup),
// the halves alternating so that no wgmma waits on the accumulator of the one just before it.  Both schedules run exactly this, so
// they give every output bit for bit the same value.  a_lo and w_lo are only read when PASSES == 3.
template <int BN, int PASSES>
__device__ __forceinline__ void mma_kblock(float* acc0, float* acc1, uint32_t a_hi, uint32_t a_lo, uint32_t w_hi, uint32_t w_lo) {
    constexpr uint32_t kHalf = 64 * 128;                        // rows 64..127 of an A box: a whole number of swizzle atoms
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) { ptx::reg_fence(acc0[i]); ptx::reg_fence(acc1[i]); }
    ptx::wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k) {
        const uint32_t koff = k * 32;   // 16 fp16 = 32 bytes inside the 128-byte swizzle row
        const uint64_t dwh = ptx::make_smem_desc_sw128(w_hi + koff);
        if (PASSES == 3) {
            const uint64_t dwl = ptx::make_smem_desc_sw128(w_lo + koff);
            wgmma_f16<BN>(acc0, ptx::make_smem_desc_sw128(a_hi + koff), dwl, 1);
            wgmma_f16<BN>(acc1, ptx::make_smem_desc_sw128(a_hi + kHalf + koff), dwl, 1);
            wgmma_f16<BN>(acc0, ptx::make_smem_desc_sw128(a_lo + koff), dwh, 1);
            wgmma_f16<BN>(acc1, ptx::make_smem_desc_sw128(a_lo + kHalf + koff), dwh, 1);
            wgmma_f16<BN>(acc0, ptx::make_smem_desc_sw128(a_hi + koff), dwh, 1);
            wgmma_f16<BN>(acc1, ptx::make_smem_desc_sw128(a_hi + kHalf + koff), dwh, 1);
        } else {
            wgmma_f16<BN>(acc0, ptx::make_smem_desc_sw128(a_hi + koff), dwh, 1);
            wgmma_f16<BN>(acc1, ptx::make_smem_desc_sw128(a_hi + kHalf + koff), dwh, 1);
        }
    }
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) { ptx::reg_fence(acc0[i]); ptx::reg_fence(acc1[i]); }
}

// Persistent schedule: gridDim.x = min(tiles, SMs); CTA b walks tiles b, b + gridDim.x, ... in m-fastest order so that concurrently
// running CTAs share the same weight columns (the W tile comes from HBM once, then from L2).
//
// Ping-pong consumers: warpgroup 1 takes the CTA's even tile ordinals, warpgroup 2 the odd ones, each with the whole 128 x BN
// accumulator.  Their main loops take turns (turn_bar), so the epilogue of tile k runs under the main loop of tile k + 1.  The ring is
// consumed in the producer's order: tile ordinal `it` starts at K-block it * kb_tile of the ring's sequence, and a warpgroup only waits
// on the ring after the other one has waited on every earlier K-block, so a parity wait never matches a phase two uses behind.
template <int BN, int PASSES, int EPI, bool TRACE = false>
__global__ void __launch_bounds__(kThreads, 1) gemm_tc_kernel(const __grid_constant__ TcParams p) {
    using Cfg = TcCfg<BN, PASSES>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::kStages * Cfg::kStageBytes);
    uint64_t* empty_bar = full_bar + Cfg::kStages;
    uint64_t* turn_bar = empty_bar + Cfg::kStages;              // [cw]: consumer warpgroup cw may start its next main loop

    const int wg = threadIdx.x >> 7;
    const int n_tiles = p.tiles_m * p.tiles_n;

    if (threadIdx.x == 0) {
        init_ring<PASSES>(p, full_bar, empty_bar, Cfg::kStages, 1);   // a slot is read by one warpgroup
        for (int c = 0; c < kConsumers; ++c) ptx::mbar_init(&turn_bar[c], 1);
        ptx::fence_mbar_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) CAPB_TRACE(0);                       // set-up done

    if (wg == 0) {
        ptx::setmaxnreg_dec<40>();
        if (threadIdx.x == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
                const int m0 = (t % p.tiles_m) * BM;
                const int n0 = (t / p.tiles_m) * BN;
                for (int s = 0; s < p.nseg; ++s) {
                    for (int kb = 0; kb < p.kblocks[s]; ++kb) {
                        ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
                        fill_stage<Cfg>(p, smem + stage * Cfg::kStageBytes, &full_bar[stage], s, kb, m0, n0);
                        if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
                    }
                }
            }
        }
    } else {
        ptx::setmaxnreg_inc<232>();
        const int cw = wg - 1;                                  // tile ordinals cw, cw + 2, ... of this CTA
        const int tid = threadIdx.x & 127;
        int kb_tile = 0;
        for (int s = 0; s < p.nseg; ++s) kb_tile += p.kblocks[s];
        int mine = 0;                                           // tiles this warpgroup has run
        for (int it = cw, t = blockIdx.x + cw * gridDim.x; t < n_tiles; it += 2, t += 2 * gridDim.x, ++mine) {
            const int m0 = (t % p.tiles_m) * BM;
            const int n0 = (t / p.tiles_m) * BN;
            // Turn: arrivals on turn_bar[cw] come from the other warpgroup at the end of ordinals cw - 1, cw + 1, ...
            if (it > 0) ptx::mbar_wait(&turn_bar[cw], (cw == 1 ? mine : mine - 1) & 1);
            if (TRACE && it == 1 && tid == 0) CAPB_TRACE(4);                           // main loop of tile 1 starts
            const long g0 = (long)it * kb_tile;
            int stage = (int)(g0 % Cfg::kStages);
            uint32_t phase = (uint32_t)(g0 / Cfg::kStages) & 1;
            float acc0[BN / 2], acc1[BN / 2];                   // rows 0..63 and 64..127 of the tile
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) { acc0[i] = 0.0f; acc1[i] = 0.0f; }
            for (int s = 0; s < p.nseg; ++s) {
                for (int kb = 0; kb < p.kblocks[s]; ++kb) {
                    ptx::mbar_wait(&full_bar[stage], phase);
                    if (TRACE && it == 0 && s == 0 && kb == 0 && tid == 0) CAPB_TRACE(1);    // first operands landed
                    const uint32_t st = ptx::smem_u32(smem + stage * Cfg::kStageBytes);
                    const uint32_t w_hi = st + Cfg::kABytes * Cfg::kPlanes;
                    mma_kblock<BN, PASSES>(acc0, acc1, st, st + Cfg::kABytes, w_hi, w_hi + Cfg::kWBytes);
                    if (tid == 0) ptx::mbar_arrive(&empty_bar[stage]);                // the slot is free again
                    if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
                }
            }
            // Every thread of the warpgroup has waited on all of this tile's K-blocks (its wgmmas, issued by all 128, retired).
            if (tid == 0) ptx::mbar_arrive(&turn_bar[cw ^ 1]);
            if (TRACE && it < 2 && tid == 0) CAPB_TRACE(2 + it);                       // main loop of tile `it` done
            epilogue_rows128<BN, EPI, TRACE>(p, acc0, acc1, m0, n0, tid, (TRACE && it < 2 && tid == 0) ? 9 + 3 * it : -1);
            if (TRACE && it < 2 && tid == 0) CAPB_TRACE(6 + it);                       // epilogue of tile `it` done
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) CAPB_TRACE(8);                       // every role is done
}

// Cooperative schedule over 256 x BN output tiles (same persistent tile walk): both consumer warpgroups read every stage, warpgroup c
// rows 128c .. 128c + 127 of the tile against the one W tile, so a K-block moves (256 + BN) rows of operands for 256 x BN outputs where
// two 128-row tiles move 2 x (128 + BN).  The main loop is bound by that feed from L2, not by the tensor cores (DESIGN §6.1).  The two
// warpgroups run their epilogues side by side, under only the producer's run-ahead into the next tile.
// TRACE slots: 1 first operands landed, 5 the producer has issued tile 0's last K-block, 2 + c / 6 + c warpgroup c's main loop /
// epilogue of tile 0 done, 9 + 3c .. 11 + 3c its LSTM stamps of rows 0..63.
template <int BN, int PASSES, int EPI, bool TRACE = false>
__global__ void __launch_bounds__(kThreads, 1) gemm_tc256_kernel(const __grid_constant__ TcParams p) {
    using Cfg = TcCfg<BN, PASSES, 2 * BM>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::kStages * Cfg::kStageBytes);
    uint64_t* empty_bar = full_bar + Cfg::kStages;

    const int wg = threadIdx.x >> 7;
    const int n_tiles = p.tiles_m * p.tiles_n;

    if (threadIdx.x == 0) {
        init_ring<PASSES>(p, full_bar, empty_bar, Cfg::kStages, kConsumers);   // a slot is read by both warpgroups
        ptx::fence_mbar_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) CAPB_TRACE(0);                       // set-up done

    if (wg == 0) {
        ptx::setmaxnreg_dec<40>();
        if (threadIdx.x == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
                const int m0 = (t % p.tiles_m) * Cfg::kTileM;
                const int n0 = (t / p.tiles_m) * BN;
                for (int s = 0; s < p.nseg; ++s) {
                    for (int kb = 0; kb < p.kblocks[s]; ++kb) {
                        ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
                        fill_stage<Cfg>(p, smem + stage * Cfg::kStageBytes, &full_bar[stage], s, kb, m0, n0);
                        if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
                    }
                }
                if (TRACE && t == (int)blockIdx.x) CAPB_TRACE(5);
            }
        }
    } else {
        ptx::setmaxnreg_inc<232>();
        const int cw = wg - 1;                                  // rows 128 cw .. 128 cw + 127 of every tile
        const int tid = threadIdx.x & 127;
        const uint32_t a_rows = cw * BM * BK * 2;               // those rows inside each A plane of a stage
        int stage = 0;
        uint32_t phase = 0;
        for (int it = 0, t = blockIdx.x; t < n_tiles; ++it, t += gridDim.x) {
            const int m0 = (t % p.tiles_m) * Cfg::kTileM + BM * cw;
            const int n0 = (t / p.tiles_m) * BN;
            float acc0[BN / 2], acc1[BN / 2];                   // rows 0..63 and 64..127 of the warpgroup's half
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) { acc0[i] = 0.0f; acc1[i] = 0.0f; }
            for (int s = 0; s < p.nseg; ++s) {
                for (int kb = 0; kb < p.kblocks[s]; ++kb) {
                    ptx::mbar_wait(&full_bar[stage], phase);
                    if (TRACE && it == 0 && s == 0 && kb == 0 && cw == 0 && tid == 0) CAPB_TRACE(1);    // first operands landed
                    const uint32_t st = ptx::smem_u32(smem + stage * Cfg::kStageBytes);
                    const uint32_t w_hi = st + Cfg::kABytes * Cfg::kPlanes;
                    mma_kblock<BN, PASSES>(acc0, acc1, st + a_rows, st + Cfg::kABytes + a_rows, w_hi, w_hi + Cfg::kWBytes);
                    if (tid == 0) ptx::mbar_arrive(&empty_bar[stage]);                // this warpgroup is done with the slot
                    if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
                }
            }
            if (TRACE && it == 0 && tid == 0) CAPB_TRACE(2 + cw);                     // main loop of tile 0 done
            epilogue_rows128<BN, EPI, TRACE>(p, acc0, acc1, m0, n0, tid, (TRACE && it == 0 && tid == 0) ? 9 + 3 * cw : -1);
            if (TRACE && it == 0 && tid == 0) CAPB_TRACE(6 + cw);                     // epilogue of tile 0 done
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

// TM = BM: the ping-pong gemm_tc_kernel; TM = 2 * BM: the cooperative gemm_tc256_kernel (BN 128 and 160 only)
template <int BN, int PASSES, int EPI, bool TRACE, int TM>
int launch_cfg(const TcParams& prm, cudaStream_t stream) {
    using Cfg = TcCfg<BN, PASSES, TM>;
    void (*kernel)(TcParams);
    if constexpr (TM == BM) kernel = gemm_tc_kernel<BN, PASSES, EPI, TRACE>;
    else kernel = gemm_tc256_kernel<BN, PASSES, EPI, TRACE>;
    static std::atomic<unsigned long long> attr_set{0};
    if (first_use_on_device(attr_set)) {
        CAPB_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
    }
    TcParams prm2 = prm;
    prm2.tiles_n = cdiv(prm.N, BN);
    prm2.tiles_m = cdiv(prm.M, TM);
    const int n_tiles = prm2.tiles_n * prm2.tiles_m;
    const int sms = sm_count();
    kernel<<<n_tiles < sms ? n_tiles : sms, kThreads, Cfg::kSmemBytes, stream>>>(prm2);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

// BN x passes of one schedule, plus the traced 3-pass kernels (capb200_decode_gemm with a trace buffer)
template <int EPI, int TM>
int launch_width(int bn, int passes, const TcParams& prm, cudaStream_t stream) {
    if (prm.trace != nullptr) {
        if (bn == 160) return launch_cfg<160, 3, EPI, true, TM>(prm, stream);
        if constexpr (TM == BM) if (bn == 64) return launch_cfg<64, 3, EPI, true, TM>(prm, stream);
        return launch_cfg<128, 3, EPI, true, TM>(prm, stream);
    }
    if (bn == 160) return passes == 3 ? launch_cfg<160, 3, EPI, false, TM>(prm, stream) : launch_cfg<160, 1, EPI, false, TM>(prm, stream);
    if constexpr (TM == BM) {
        if (bn == 64) return passes == 3 ? launch_cfg<64, 3, EPI, false, TM>(prm, stream) : launch_cfg<64, 1, EPI, false, TM>(prm, stream);
    }
    return passes == 3 ? launch_cfg<128, 3, EPI, false, TM>(prm, stream) : launch_cfg<128, 1, EPI, false, TM>(prm, stream);
}

template <int EPI>
int launch_kind(int bm, int bn, int passes, const TcParams& prm, cudaStream_t stream) {
    return bm == 2 * BM ? launch_width<EPI, 2 * BM>(bn, passes, prm, stream) : launch_width<EPI, BM>(bn, passes, prm, stream);
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

// Tile height of one launch: M rows (the launch's own, which may be fewer than the plan's) on a plan of width bn.  The main loop is fed,
// not computed (DESIGN §6.1): a K-block moves (BM + BN) rows of operands into a CTA, so 256-row tiles move 28 % (BN 160) or 25 %
// (BN 128) fewer bytes per output than 128-row ones.  But the cooperative schedule exposes the epilogue of every tile a CTA runs, where
// the ping-pong one exposes only the last.  So 256 rows are taken where they fit the launch in one wave and 128 rows would need more:
// there both expose one epilogue per CTA (the 1280 x 4000 LSTM gates of the decode step).  Where 256-row tiles take several waves (logit,
// att_embed) or 128-row ones already take one (the t = 0 gate launches of 256 rows, the few-row baseline launches), the ping-pong
// schedule measured faster (tools/decode_gemm_rate.py, DESIGN §6.1).  BN 64 has no 256-row kernel.  CAPB200_GEMM_BM=128 or 256 forces
// a height for A/B timing and tests; it is read at every call, so a process can switch it between launches.
int gemm_tc_tile_m(int M, int N, int bn) {
    if (bn == 64) return BM;
    const char* force = getenv("CAPB200_GEMM_BM");
    if (force != nullptr && strcmp(force, "128") == 0) return BM;
    if (force != nullptr && strcmp(force, "256") == 0) return 2 * BM;
    const int sms = sm_count();
    const int tiles_n = cdiv(N, bn);
    return cdiv(M, 2 * BM) * tiles_n <= sms && cdiv(M, BM) * tiles_n > sms ? 2 * BM : BM;
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
    if (M_override > plan->prm.M) { set_error("gemm_tc: M override exceeds the planned row count"); return 1; }
    const int M = M_override > 0 ? M_override : plan->prm.M;
    TcParams prm = plan->prm;
    if (epi_override != nullptr) fill_epilogue(prm, *epi_override);
    prm.M = M;
    if (prm.lstm && (prm.N != 4 * prm.H || prm.c_out == nullptr || prm.h_f == nullptr)) {
        set_error("gemm_tc: fused LSTM epilogue needs N == 4H, c_out and h_f");
        return 1;
    }
    if (prm.M <= 0 || prm.N <= 0) return 0;
    // the kind follows the epilogue this launch asks for: launches override the planned one whole
    const int kind = prm.lstm ? kEpiLstm : prm.C_hi != nullptr ? kEpiPlanes : kEpiStore;
    if (prm.trace != nullptr && plan->passes != 3) { set_error("gemm_tc: the traced kernel is the 3-pass one"); return 1; }
    const int bm = gemm_tc_tile_m(prm.M, prm.N, plan->bn);            // per launch: M may be fewer rows than planned
    if (kind == kEpiLstm) return launch_kind<kEpiLstm>(bm, plan->bn, plan->passes, prm, stream);
    if (kind == kEpiPlanes) return launch_kind<kEpiPlanes>(bm, plan->bn, plan->passes, prm, stream);
    return launch_kind<kEpiStore>(bm, plan->bn, plan->passes, prm, stream);
}

}  // namespace capb200
