// wgmma tf32 GEMM for the training steps (SCST / XE):  C[M,N] (+)= sum_s X_s[M,K_s] * W_s[N,K_s]^T (+ bias + row bias)
//
// Replaces the mma.sync 3xTF32 kernels of gemm_generic.cu on the hot path of LossWrapper's sc branch (reference call sites:
// captioning/modules/loss_wrapper.py:56-73 -> every nn.Linear / nn.LSTMCell of AoAModel.py / AttModel.py in train mode, and the
// input-gradient / weight-gradient contractions autograd runs for them in loss.backward(), tools/train.py:189).
//
// Numerics.  The training steps read the fp32 parameters in place (they change every optimizer step) and multiply gradient rows of
// ~1e-7, which fp16 planes would flush to zero, so the operands stay fp32 in HBM and are split INSIDE the kernel into TF32 pairs:
//   hi = cvt.rna.tf32(x)  (exactly representable: the tensor core's own fp32 -> tf32 conversion, whatever its rounding, is the identity)
//   lo = x - hi           (exact in fp32; the tensor core keeps its top 11 bits: relative error <= 2^-21 of x)
// and every K-block issues three tf32 wgmmas into one fp32 register accumulator: hi*lo + lo*hi + hi*hi (3xTF32, dropped lo*lo <= 2^-22).
//
// Structure (one 128 x BN accumulator tile per CTA, 384 threads = three warpgroups, split-K across a thread-block cluster):
//   warpgroup 0     TMA producer (one thread): cp.async.bulk.tensor 2-D boxes of RAW fp32 [32 k x 128 rows] (A side) and [32 k x BN rows]
//                   (B side), 128B swizzle, into a STAGES-deep ring (mbarrier complete_tx).
//   warpgroups 1,2  converters and MMA issuers: read the raw tiles from shared memory, write hi in place and lo next to it (element-wise,
//                   so the swizzle pattern is preserved), fence.proxy.async, meet at a named barrier, then each issues the wgmmas of its
//                   64 accumulator rows (m64nNk8) and releases the slot once they retired.
//   epilogue        the consumers drain the register accumulators into a shared-memory staging tile laid out like the OUTPUT (so global
//                   stores are coalesced); with split-K the CTAs of the cluster (cluster dim = ksplit <= 8, K-ranges side by side) then
//                   add their tiles through distributed shared memory in rank order (deterministic, no atomics, no second kernel) and
//                   each stores a slice.
// Operand roles: the A side always supplies 128 accumulator rows, the B side BN columns.  Skinny problems (M <= 256 activation rows:
// the 50-row sampling steps) run SWAPPED -- weights on the A side, activations on the B side -- so no tensor-core row is padding and
// the weights are streamed exactly once; problems with many rows (refiner: B*R rows; batched-over-time gradients: T*N rows) run normally.
#include <cstring>
#include <mutex>
#include <unordered_map>

#include "common.cuh"
#include "kernels.cuh"
#include "ptx.cuh"

namespace capb200 {

namespace {

constexpr int TM = 128;          // accumulator rows per CTA (A-side rows)
constexpr int TK = 32;           // fp32 elements per K-block: one 128-byte swizzle row
constexpr int kMaxSegT = 3;
constexpr int kConvThreads = 256;   // warpgroups 1 and 2
constexpr int kConsumersT = 2;
constexpr int kThreadsT = 128 + kConvThreads;

struct Tf32Params {
    CUtensorMap a_map[kMaxSegT];
    CUtensorMap b_map[kMaxSegT];
    int kblocks[kMaxSegT];
    int nseg;
    int ksteps_total;
    int swapped;                  // 1: A side = weights (output columns), B side = activations (output rows)
    int M, N;                     // output extents
    float* C;
    long ldc;
    const float* bias;            // [N]
    const float* row_bias;        // [M / rpg, N]
    long ld_rb;
    int rpg;
    int accumulate;
    // split-K without a cluster (finer splits than 8, no co-scheduling constraint): every K-rank writes its tile to `scratch`, the last CTA
    // of a tile to arrive (per-tile counter) adds the ranks in rank order -- deterministic -- and applies the epilogue.  nullptr = cluster / DSMEM (the default; see gemm_tf32_launch).
    float* scratch;
    unsigned int* counters;
};

template <int BN>
struct Tf32Cfg {
    static constexpr uint32_t kABytes = TM * TK * 4;                 // 16 KB
    static constexpr uint32_t kBBytes = BN * TK * 4;
    static constexpr uint32_t kStageBytes = 2 * (kABytes + kBBytes);  // raw->hi and lo copies of both tiles
    static constexpr int kStages = (192 * 1024) / kStageBytes >= 6 ? 6 : (192 * 1024) / kStageBytes;
    static constexpr uint32_t kRingBytes = kStages * kStageBytes;
    static constexpr int kPad = 4;
    // staging tile in OUTPUT orientation: swapped -> [BN rows(m)][128 + pad]; normal -> [128 rows(m)][BN + pad]; aliases the ring
    static constexpr uint32_t kStagingSwapped = BN * (TM + kPad) * 4;
    static constexpr uint32_t kStagingNormal = TM * (BN + kPad) * 4;
    static constexpr uint32_t kStaging = kStagingSwapped > kStagingNormal ? kStagingSwapped : kStagingNormal;
    static constexpr uint32_t kBody = kRingBytes > kStaging ? kRingBytes : kStaging;
    static constexpr uint32_t kSmemBytes = kBody + 1024 /*align*/ + 512 /*barriers*/;
    static_assert(BN == 32 || BN == 64 || BN == 128 || BN == 256, "wgmma wrappers exist for N = 32, 64, 128 (256 = two halves)");
    static_assert(kStages >= 2, "need a double buffer");
    static_assert(kBBytes % 1024 == 0, "tiles must keep the 1024-byte swizzle-atom alignment");
    static_assert(kSmemBytes <= 227 * 1024, "shared memory of one H100 block");
};

// acc[BN / 2] (+)= A[64 rows] * B[BN rows]^T for one k8 step; N = 256 runs as two N = 128 halves (B rows 128.. start 16 KB further)
template <int BN>
__device__ __forceinline__ void wgmma_tf32(float* acc, uint32_t a, uint32_t b) {
    const uint64_t da = ptx::make_smem_desc_sw128(a);
    if (BN == 32) ptx::wgmma_tf32_n32(acc, da, ptx::make_smem_desc_sw128(b), 1);
    else if (BN == 64) ptx::wgmma_tf32_n64(acc, da, ptx::make_smem_desc_sw128(b), 1);
    else {
#pragma unroll
        for (int h = 0; h < BN / 128; ++h) ptx::wgmma_tf32_n128(acc + 64 * h, da, ptx::make_smem_desc_sw128(b + h * 128 * 128), 1);
    }
}

__device__ __forceinline__ uint32_t mapa_shared(uint32_t addr, uint32_t rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
    return r;
}
__device__ __forceinline__ float4 ld_dsmem_f4(uint32_t addr) {
    float4 v;
    asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
    return v;
}
// the 256 converter / consumer threads only (the producer warpgroup never joins)
__device__ __forceinline__ void consumers_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kConvThreads) : "memory"); }

__device__ __forceinline__ void split_keep_tf32(float x, float& hi, float& lo) {
    uint32_t h;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(h) : "f"(x));
    hi = __uint_as_float(h);
    lo = x - hi;
}

template <int BN>
__global__ void __launch_bounds__(kThreadsT, 1) gemm_tf32x3_kernel(const __grid_constant__ Tf32Params p) {
    using Cfg = Tf32Cfg<BN>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::kBody);
    uint64_t* empty_bar = full_bar + Cfg::kStages;

    const int wg = threadIdx.x >> 7;
    const int ksplit = gridDim.x;                       // cluster = (ksplit, 1, 1): blockIdx.x is the K-rank
    const int krank = blockIdx.x;
    const int a_row0 = blockIdx.y * TM;                 // first A-side row of this tile
    const int b_row0 = blockIdx.z * BN;                 // first B-side row
    const int ks0 = (int)(((long)p.ksteps_total * krank) / ksplit);
    const int ks1 = (int)(((long)p.ksteps_total * (krank + 1)) / ksplit);
    const int nk = ks1 - ks0;

    if (threadIdx.x == 0) {
        for (int s = 0; s < p.nseg; ++s) { ptx::prefetch_tmap(&p.a_map[s]); ptx::prefetch_tmap(&p.b_map[s]); }
        for (int i = 0; i < Cfg::kStages; ++i) {
            ptx::mbar_init(&full_bar[i], 1);
            ptx::mbar_init(&empty_bar[i], kConsumersT);
        }
        ptx::fence_mbar_init();
    }
    __syncthreads();

    // flattened K-step -> (segment, k-block inside the segment)
    auto locate = [&](int ks, int& seg, int& kb) {
        seg = 0;
        int first = 0;
        while (seg < p.nseg - 1 && ks >= first + p.kblocks[seg]) { first += p.kblocks[seg]; ++seg; }
        kb = ks - first;
    };

    if (wg == 0) {
        if (threadIdx.x == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int it = 0; it < nk; ++it) {
                int seg, kb;
                locate(ks0 + it, seg, kb);
                ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
                uint8_t* st = smem + stage * Cfg::kStageBytes;
                ptx::mbar_arrive_expect_tx(&full_bar[stage], Cfg::kABytes + Cfg::kBBytes);
                ptx::tma_load_2d(st, &p.a_map[seg], &full_bar[stage], kb * TK, a_row0);
                ptx::tma_load_2d(st + 2 * Cfg::kABytes, &p.b_map[seg], &full_bar[stage], kb * TK, b_row0);
                if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
            }
        }
    } else {
        const int ct = threadIdx.x - 128;               // 0 .. 255 over both consumer warpgroups
        const int cw = wg - 1;                          // accumulator rows [64 cw, 64 cw + 64) of the tile
        const int tid = threadIdx.x & 127;
        float acc[BN / 2];
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0.0f;
        int stage = 0;
        uint32_t phase = 0;
        constexpr int kAVec = Cfg::kABytes / 16, kBVec = Cfg::kBBytes / 16;
        for (int it = 0; it < nk; ++it) {
            ptx::mbar_wait(&full_bar[stage], phase);
            // ---- converters: raw fp32 -> (hi in place, lo beside it); purely element-wise, so the TMA swizzle is preserved
            uint8_t* st = smem + stage * Cfg::kStageBytes;
            float4* a_hi = reinterpret_cast<float4*>(st);
            float4* a_lo = reinterpret_cast<float4*>(st + Cfg::kABytes);
            float4* b_hi = reinterpret_cast<float4*>(st + 2 * Cfg::kABytes);
            float4* b_lo = reinterpret_cast<float4*>(st + 2 * Cfg::kABytes + Cfg::kBBytes);
#pragma unroll 4
            for (int i = ct; i < kAVec; i += kConvThreads) {
                const float4 x = a_hi[i];
                float4 h, l;
                split_keep_tf32(x.x, h.x, l.x); split_keep_tf32(x.y, h.y, l.y); split_keep_tf32(x.z, h.z, l.z); split_keep_tf32(x.w, h.w, l.w);
                a_hi[i] = h;
                a_lo[i] = l;
            }
#pragma unroll 4
            for (int i = ct; i < kBVec; i += kConvThreads) {
                const float4 x = b_hi[i];
                float4 h, l;
                split_keep_tf32(x.x, h.x, l.x); split_keep_tf32(x.y, h.y, l.y); split_keep_tf32(x.z, h.z, l.z); split_keep_tf32(x.w, h.w, l.w);
                b_hi[i] = h;
                b_lo[i] = l;
            }
            ptx::fence_proxy_async_smem();              // generic-proxy writes -> visible to the tensor core's async-proxy reads
            consumers_sync();                           // both warpgroups' halves of the conversion are done
            const uint32_t s0 = ptx::smem_u32(st);
            const uint32_t ah = s0 + cw * 64 * 128, al = s0 + Cfg::kABytes + cw * 64 * 128;
            const uint32_t bh = s0 + 2 * Cfg::kABytes, bl = bh + Cfg::kBBytes;
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) ptx::reg_fence(acc[i]);
            ptx::wgmma_fence();
#pragma unroll
            for (int k = 0; k < TK / 8; ++k) {
                const uint32_t koff = k * 32;          // 8 tf32 = 32 bytes inside the 128-byte swizzle row
                wgmma_tf32<BN>(acc, ah + koff, bl + koff);
                wgmma_tf32<BN>(acc, al + koff, bh + koff);
                wgmma_tf32<BN>(acc, ah + koff, bh + koff);
            }
            ptx::wgmma_commit();
            ptx::wgmma_wait<0>();
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) ptx::reg_fence(acc[i]);
            if (tid == 0) ptx::mbar_arrive(&empty_bar[stage]);
            if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
        }
        // ---- drain the accumulator into the staging tile (output orientation); it aliases the ring, so both warpgroups' wgmmas must
        // have retired first (the producer's loads all landed: every one of them was waited for above)
        consumers_sync();
        float* S = reinterpret_cast<float*>(smem);
        const int warp = tid >> 5, lane = tid & 31;
        const int arow0 = cw * 64 + warp * 16 + (lane >> 2);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int arow = arow0 + 8 * (e >> 1);
                const int bcol = 8 * j + 2 * (lane & 3) + (e & 1);
                if (p.swapped) S[bcol * (TM + Cfg::kPad) + arow] = acc[4 * j + e];
                else S[arow * (BN + Cfg::kPad) + bcol] = acc[4 * j + e];
            }
        }
    }
    __syncthreads();
    const bool via_scratch = ksplit > 1 && p.scratch != nullptr;
    if (ksplit > 1 && !via_scratch) ptx::cluster_sync_all();            // every K-rank's staging tile is complete and visible cluster-wide

    // ---- reduce across the K-ranks (fixed order) and store
    {
        const int rows_out = p.swapped ? BN : TM;
        const int cols_out = p.swapped ? TM : BN;
        const int pitch = cols_out + Cfg::kPad;
        const int vec_per_row = cols_out / 4;
        const int tile_vecs = rows_out * vec_per_row;
        int r_lo = rows_out * krank / ksplit, r_hi = rows_out * (krank + 1) / ksplit;      // cluster form: rank r owns a slice of the tile's rows
        const float4* part = nullptr;
        bool active = true;
        if (via_scratch) {
            __shared__ int s_last;
            const long tile_id = (long)blockIdx.y * gridDim.z + blockIdx.z;
            float4* mine = reinterpret_cast<float4*>(p.scratch) + (tile_id * ksplit + krank) * tile_vecs;
            for (int idx = threadIdx.x; idx < tile_vecs; idx += kThreadsT) {
                const int ro = idx / vec_per_row, co = (idx % vec_per_row) * 4;
                __stcg(mine + idx, *reinterpret_cast<const float4*>(smem + (ro * pitch + co) * 4));
            }
            __threadfence();
            __syncthreads();
            if (threadIdx.x == 0) s_last = (atomicAdd(p.counters + tile_id, 1u) == (unsigned)(ksplit - 1)) ? 1 : 0;
            __syncthreads();
            active = s_last != 0;                                   // the last K-rank to arrive finishes the tile
            if (active) {
                __threadfence();
                if (threadIdx.x == 0) p.counters[tile_id] = 0u;     // ready for the next launch (stream order)
                part = reinterpret_cast<const float4*>(p.scratch) + tile_id * ksplit * tile_vecs;
                r_lo = 0; r_hi = rows_out;
            }
        }
        const int m_base = p.swapped ? b_row0 : a_row0;
        const int n_base = p.swapped ? a_row0 : b_row0;
        const uint32_t s_base = ptx::smem_u32(smem);
        const bool vec_ok = (p.ldc & 3) == 0 && (reinterpret_cast<uintptr_t>(p.C) & 15) == 0 && (n_base & 3) == 0;
        for (int idx = threadIdx.x; active && idx < (r_hi - r_lo) * vec_per_row; idx += kThreadsT) {
            const int ro = r_lo + idx / vec_per_row, co = (idx % vec_per_row) * 4;
            const int m = m_base + ro, n = n_base + co;
            if (m >= p.M || n >= p.N) continue;
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            const uint32_t off = s_base + static_cast<uint32_t>((ro * pitch + co) * 4);
            if (ksplit == 1) {
                acc = *reinterpret_cast<const float4*>(smem + (ro * pitch + co) * 4);
            } else if (via_scratch) {
                for (int kr = 0; kr < ksplit; ++kr) {
                    const float4 v = __ldcg(part + (long)kr * tile_vecs + ro * vec_per_row + co / 4);
                    acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
                }
            } else {
                for (int kr = 0; kr < ksplit; ++kr) {
                    const float4 v = ld_dsmem_f4(mapa_shared(off, (uint32_t)kr));
                    acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
                }
            }
            float v[4] = {acc.x, acc.y, acc.z, acc.w};
            const float* rb = p.row_bias ? p.row_bias + (long)(m / p.rpg) * p.ld_rb : nullptr;
            float* c = p.C + (long)m * p.ldc + n;
            if (n + 4 <= p.N && vec_ok) {
                if (p.bias) { v[0] += __ldg(p.bias + n); v[1] += __ldg(p.bias + n + 1); v[2] += __ldg(p.bias + n + 2); v[3] += __ldg(p.bias + n + 3); }
                if (rb) { v[0] += __ldg(rb + n); v[1] += __ldg(rb + n + 1); v[2] += __ldg(rb + n + 2); v[3] += __ldg(rb + n + 3); }
                if (p.accumulate) { const float4 o = *reinterpret_cast<const float4*>(c); v[0] += o.x; v[1] += o.y; v[2] += o.z; v[3] += o.w; }
                *reinterpret_cast<float4*>(c) = make_float4(v[0], v[1], v[2], v[3]);
            } else {
                for (int u = 0; u < 4; ++u) {
                    if (n + u >= p.N) break;
                    float x = v[u];
                    if (p.bias) x += __ldg(p.bias + n + u);
                    if (rb) x += __ldg(rb + n + u);
                    if (p.accumulate) x += c[u];
                    c[u] = x;
                }
            }
        }
    }
    __syncthreads();
    if (ksplit > 1 && !via_scratch) ptx::cluster_sync_all();            // nobody leaves while a peer may still read its staging tile
}

// ---- transposes for operands that are not K-major in HBM (input gradients need W^T, weight gradients dY^T and X^T) -------------------
__global__ void transpose_kernel(const float* __restrict__ src, long ld_src, int rows, int cols, float* __restrict__ dst, long ld_dst) {
    __shared__ float tile[32][33];
    const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
    for (int i = threadIdx.y; i < 32; i += 8) {
        const int r = r0 + i, c = c0 + threadIdx.x;
        tile[i][threadIdx.x] = (r < rows && c < cols) ? src[(long)r * ld_src + c] : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += 8) {
        const int c = c0 + i, r = r0 + threadIdx.x;           // dst[c][r]
        if (c < cols && r < rows) dst[(long)c * ld_dst + r] = tile[threadIdx.x][i];
    }
}

// ---- host side -------------------------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (fn == nullptr) {
        void* sym = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres) != cudaSuccess || sym == nullptr) return nullptr;
        fn = reinterpret_cast<EncodeTiledFn>(sym);
    }
    return fn;
}

struct MapKey {
    const void* base; long rows, K, pitch; int box_rows;
    bool operator==(const MapKey& o) const { return base == o.base && rows == o.rows && K == o.K && pitch == o.pitch && box_rows == o.box_rows; }
};
struct MapKeyHash {
    size_t operator()(const MapKey& k) const {
        size_t h = reinterpret_cast<size_t>(k.base);
        h ^= (size_t)k.rows * 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2);
        h ^= (size_t)k.K * 0xC2B2AE3D27D4EB4Full + (h << 6) + (h >> 2);
        h ^= (size_t)k.pitch * 0x165667B19E3779F9ull + (h << 6) + (h >> 2);
        return h ^ (size_t)k.box_rows;
    }
};

}  // namespace

// Encoded-tensor-map cache + transposed-operand cache of one engine (training buffers are stable across steps, so after the first step
// every lookup hits).  Not thread-safe by itself: one context per engine, engines are not re-entrant (include/capb200.h).
struct Tf32Context {
    std::unordered_map<MapKey, CUtensorMap, MapKeyHash> maps;
    struct TEntry { float* buf = nullptr; size_t floats = 0; unsigned long long stamp = 0; };
    std::unordered_map<MapKey, TEntry, MapKeyHash> transposed;        // key: (src, rows, cols, ld_src)
    unsigned long long stamp = 1;                                      // bumped per training step: weight transposes are rebuilt once per step
    long launches = 0;
    float* scratch = nullptr;          // split-K partial tiles [tile][K-rank][rows][cols]
    size_t scratch_floats = 0;
    unsigned int* counters = nullptr;  // per-tile arrival counters (zero between launches)
    int n_counters = 0;
};

Tf32Context* tf32_context_create() { return new Tf32Context(); }
void tf32_context_destroy(Tf32Context* c) {
    if (c == nullptr) return;
    for (auto& kv : c->transposed) cudaFree(kv.second.buf);
    cudaFree(c->scratch);
    cudaFree(c->counters);
    delete c;
}
void tf32_context_new_step(Tf32Context* c) { if (c) c->stamp++; }
long tf32_context_launches(const Tf32Context* c) { return c ? c->launches : 0; }

namespace {

const CUtensorMap* get_map(Tf32Context* ctx, const float* base, long rows, long K, long pitch, int box_rows, std::string* err) {
    const MapKey key{base, rows, K, pitch, box_rows};
    auto it = ctx->maps.find(key);
    if (it != ctx->maps.end()) return &it->second;
    EncodeTiledFn fn = encode_fn();
    if (fn == nullptr) { *err = "cuTensorMapEncodeTiled entry point not available"; return nullptr; }
    CUtensorMap m;
    cuuint64_t gdim[2] = {static_cast<cuuint64_t>(K), static_cast<cuuint64_t>(rows)};
    cuuint64_t gstride[1] = {static_cast<cuuint64_t>(pitch) * 4};
    cuuint32_t box[2] = {static_cast<cuuint32_t>(TK), static_cast<cuuint32_t>(box_rows)};
    cuuint32_t estr[2] = {1, 1};
    const CUresult r = fn(&m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                          CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { *err = "cuTensorMapEncodeTiled(fp32) failed with CUresult " + std::to_string((int)r); return nullptr; }
    return &(ctx->maps[key] = m);
}

template <int BN>
int launch_tf32(const Tf32Params& prm, int ksplit, int tiles_a, int tiles_b, cudaStream_t st) {
    using Cfg = Tf32Cfg<BN>;
    static std::atomic<unsigned long long> attr_set{0};
    if (first_use_on_device(attr_set)) {
        CAPB_CHECK_CUDA(cudaFuncSetAttribute(gemm_tf32x3_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(ksplit, tiles_a, tiles_b);
    cfg.blockDim = dim3(kThreadsT);
    cfg.dynamicSmemBytes = Cfg::kSmemBytes;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = ksplit;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = (ksplit > 1 && prm.scratch == nullptr) ? 1 : 0;
    CAPB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, gemm_tf32x3_kernel<BN>, prm));
    return 0;
}

bool tma_ok(const float* p, long pitch, int K) { return p != nullptr && (reinterpret_cast<uintptr_t>(p) & 15) == 0 && (pitch & 3) == 0 && K >= 1; }

}  // namespace

bool gemm_tf32_supported(int nseg, const float* const* X, const long* ldx, const float* const* W, const long* ldw, const int* K) {
    if (nseg < 1 || nseg > kMaxSegT) return false;
    for (int s = 0; s < nseg; ++s)
        if (!tma_ok(X[s], ldx[s], K[s]) || !tma_ok(W[s], ldw[s], K[s])) return false;
    return true;
}

// C[M,N] (+)= sum_s X_s[M,K_s] * W_s[N,K_s]^T (+ bias[N] + row_bias[m / rpg, N]); every operand K-major (row-major [rows, K]) fp32 with
// 16-byte aligned rows.  Returns 0, or 1 with last_error set.
int gemm_tf32_launch(Tf32Context* ctx, int M, int N, int nseg, const float* const* X, const long* ldx, const float* const* W, const long* ldw, const int* K,
                     float* C, long ldc, const float* bias, const float* row_bias, long ld_rb, int rpg, int accumulate, cudaStream_t st) {
    if (M <= 0 || N <= 0) return 0;
    CAPB_REQUIRE(ctx != nullptr, "gemm_tf32: no context");
    CAPB_REQUIRE(gemm_tf32_supported(nseg, X, ldx, W, ldw, K), "gemm_tf32: operands must be fp32, K-major, 16-byte aligned rows, 1..3 segments");
    Tf32Params p;
    memset(&p, 0, sizeof(p));
    p.nseg = nseg; p.M = M; p.N = N; p.C = C; p.ldc = ldc; p.bias = bias; p.row_bias = row_bias; p.ld_rb = ld_rb; p.rpg = rpg < 1 ? 1 : rpg;
    p.accumulate = accumulate;
    const bool swapped = M <= 256;
    p.swapped = swapped ? 1 : 0;
    int bn;
    if (swapped) bn = M <= 32 ? 32 : M <= 64 ? 64 : M <= 128 ? 128 : 256;
    else bn = 128;
    const long a_rows = swapped ? N : M, b_rows = swapped ? M : N;
    int ksteps = 0;
    std::string err;
    for (int s = 0; s < nseg; ++s) {
        const float* a_base = swapped ? W[s] : X[s];
        const float* b_base = swapped ? X[s] : W[s];
        const long a_pitch = swapped ? ldw[s] : ldx[s], b_pitch = swapped ? ldx[s] : ldw[s];
        const CUtensorMap* ma = get_map(ctx, a_base, a_rows, K[s], a_pitch, TM, &err);
        const CUtensorMap* mb = ma ? get_map(ctx, b_base, b_rows, K[s], b_pitch, bn, &err) : nullptr;
        if (ma == nullptr || mb == nullptr) { set_error("gemm_tf32: " + err); return 1; }
        p.a_map[s] = *ma;
        p.b_map[s] = *mb;
        p.kblocks[s] = cdiv(K[s], TK);
        ksteps += p.kblocks[s];
    }
    p.ksteps_total = ksteps;
    const int tiles_a = (int)cdiv((int)a_rows, TM), tiles_b = (int)cdiv((int)b_rows, bn);
    // split-K so that ~all SMs stream disjoint K-slices.
    //  * across a thread-block cluster with the DSMEM reduction (largest power of two <= 8 with tiles * ksplit <= SMs), except for the
    //    shape class named below.
    //  * 16 or more clusters of 8 (att2ctx and its input gradient, 2048 x 2048): finer splits (up to 24 K-ranks, >= 2 K-blocks each) with
    //    the partial tiles in a global scratch buffer and a last-arriver reduction in rank order.  The scratch form wins where the cluster
    //    form tops out on a large K, and loses elsewhere, where the last CTA re-reads many partial tiles.
    const long tiles = (long)tiles_a * tiles_b;
    const int sms = sm_count();
    int ksplit = 1;
    while (ksplit < 8 && tiles * (ksplit * 2) <= sms && ksteps / (ksplit * 2) >= 2) ksplit *= 2;
    const bool use_scratch = ksplit == 8 && tiles >= 16;
    if (use_scratch) {
        ksplit = (int)(sms / tiles);
        if (ksplit > ksteps / 2) ksplit = ksteps / 2;
        if (ksplit > 24) ksplit = 24;
        if (ksplit < 1) ksplit = 1;
        if (ksplit > 1) {
            const size_t need = (size_t)tiles * ksplit * TM * bn;
            if (need > ctx->scratch_floats || tiles > ctx->n_counters) {
                CAPB_CHECK_CUDA(cudaStreamSynchronize(st));
                if (need > ctx->scratch_floats) {
                    if (ctx->scratch) CAPB_CHECK_CUDA(cudaFree(ctx->scratch));
                    ctx->scratch = nullptr;
                    const size_t grow = need > ((size_t)8 << 20) ? need : ((size_t)8 << 20);
                    CAPB_CHECK_CUDA(cudaMalloc(&ctx->scratch, grow * sizeof(float)));
                    ctx->scratch_floats = grow;
                }
                if (tiles > ctx->n_counters) {
                    if (ctx->counters) CAPB_CHECK_CUDA(cudaFree(ctx->counters));
                    ctx->counters = nullptr;
                    const int nc = tiles > 4096 ? (int)tiles : 4096;
                    CAPB_CHECK_CUDA(cudaMalloc(&ctx->counters, nc * sizeof(unsigned int)));
                    CAPB_CHECK_CUDA(cudaMemsetAsync(ctx->counters, 0, nc * sizeof(unsigned int), st));
                    ctx->n_counters = nc;
                }
            }
            p.scratch = ctx->scratch;
            p.counters = ctx->counters;
        }
    }
    ctx->launches++;
    switch (bn) {
        case 32: return launch_tf32<32>(p, ksplit, tiles_a, tiles_b, st);
        case 64: return launch_tf32<64>(p, ksplit, tiles_a, tiles_b, st);
        case 128: return launch_tf32<128>(p, ksplit, tiles_a, tiles_b, st);
        default: return launch_tf32<256>(p, ksplit, tiles_a, tiles_b, st);
    }
}

// dst[cols, rows] = src[rows, cols]^T into a context-owned buffer.  `per_step` entries (weights) are rebuilt once per training step
// (tf32_context_new_step), the others (activations / gradients of the step) on every call.
const float* tf32_transposed(Tf32Context* ctx, const float* src, long ld_src, int rows, int cols, bool per_step, long* ld_dst, cudaStream_t st) {
    const MapKey key{src, rows, cols, ld_src, per_step ? 1 : 0};
    Tf32Context::TEntry& e = ctx->transposed[key];
    const long ld = round_up(rows, 4);
    const size_t need = (size_t)cols * ld;
    if (e.floats < need) {
        if (e.buf) cudaFree(e.buf);
        e.buf = nullptr;
        if (cudaMalloc(&e.buf, need * sizeof(float)) != cudaSuccess) { set_error("gemm_tf32: out of memory for a transposed operand"); return nullptr; }
        if (cudaMemsetAsync(e.buf, 0, need * sizeof(float), st) != cudaSuccess) return nullptr;
        e.floats = need;
        e.stamp = 0;
    }
    *ld_dst = ld;
    if (per_step && e.stamp == ctx->stamp) return e.buf;
    dim3 grid(cdiv(cols, 32), cdiv(rows, 32));
    transpose_kernel<<<grid, dim3(32, 8), 0, st>>>(src, ld_src, rows, cols, e.buf, ld);
    if (cudaGetLastError() != cudaSuccess) { set_error("gemm_tf32: transpose launch failed"); return nullptr; }
    ctx->launches++;
    e.stamp = ctx->stamp;
    return e.buf;
}

}  // namespace capb200
