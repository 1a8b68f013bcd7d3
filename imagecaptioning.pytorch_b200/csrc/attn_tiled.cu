// Key-tiled multi-head attention: the forms of the refiner / encoder self-attention, of the Transformer decoder's causal self-attention and of
// the decoder's cross-attention backward that the staged kernels (transformer.cu, aoa_train_kernels.cu) cannot hold in 200 KB of shared
// memory.  K, V and the scores stream through shared memory one tile of 32 keys at a time, so no shared-memory footprint grows with the
// region count or the caption length.  Causal (key r visible to query i iff r <= i): the key tiles past a query tile's last query are
// skipped, and the tile that straddles the diagonal masks the keys past each query.
//
//   forward        one CTA per (sequence, head, tile of 32 queries); online softmax over the key tiles, key mask (-inf) and the
//                  replayable probability dropout (p = 0: the decode form)
//   backward       the FlashAttention-2 structure without float atomics (bitwise reproducible):
//     row pass     per query: softmax statistics (self) and delta_i = sum_r P_ir Z_ir (dO_i . V_r)   (Z = dropout scale)
//     dK / dV      one CTA per key tile walks the query tiles
//     dQ           one CTA per query tile walks the key tiles
//   The backward keeps no workspace: the row pass writes each (row, head)'s statistics into the first three columns of that row's dq head
//   slice, the dK / dV pass reads them there, and the dQ pass reads its own rows' statistics before it overwrites them.  dq therefore must
//   not alias q, k, v or d_out.
//
// Dropout element indices are those of the staged kernels, so capb200_dropout_mask replays the masks unchanged:
//   self-attention   ((b * heads + head) * idx_L + qi) * idx_L + r, step 0
//   cross-attention  item_local * R + r with item_local = (image row within the time block) * heads + head, step = step + time block
#include "common.cuh"
#include "dropout.cuh"
#include "kernels.cuh"

namespace capb200 {

namespace {

constexpr int kTile = 32;           // keys per key tile (one per lane) and queries per query tile
constexpr int kThreads = 256;
constexpr int kPerWarp = kTile / (kThreads / 32);       // queries (or keys) a warp owns inside a tile

__device__ __forceinline__ float t_wsum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float t_wmax(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float t_dot(const float* __restrict__ a, const float* __restrict__ b, int dk4) {
    const float4* a4 = reinterpret_cast<const float4*>(a);
    const float4* b4 = reinterpret_cast<const float4*>(b);
    float s = 0.f;
    for (int c = 0; c < dk4; ++c) {
        const float4 x = a4[c], y = b4[c];
        s = fmaf(x.x, y.x, fmaf(x.y, y.y, fmaf(x.z, y.z, fmaf(x.w, y.w, s))));
    }
    return s;
}

// Queries i of sequence s (image-major self-attention: row = s * q_seq + i * q_pos; cross-attention rows are TIME-major blocks of q_blk rows
// per image: row = (i / q_blk) * q_blk_stride + s * q_seq + (i % q_blk) * q_pos), keys r of sequence s at row s * k_seq + r * k_pos.
struct TiledAttn {
    int nq, nk, dk, heads;
    int q_blk;
    long q_blk_stride, q_seq, q_pos, k_seq, k_pos;
    const float *q, *k, *v, *d_out;
    float *dq, *dk_, *dv;
    long ld_q, ld_kv, ld_do, ld_dq, ld_dkv;
    float scale, p_drop;
    unsigned long long seed;
    uint32_t site, step;
    int cross, idx_L;
    int causal, q_lo;               // causal self-attention; forward: the queries are [q_lo, nq)
    const float* key_mask;          // self-attention: [seqs, ld_mask], 0 = masked key
    long ld_mask;
    const float* probs;             // cross-attention: saved probabilities [(row * heads + head) * nk + r]

    __device__ long q_row(int s, int i) const { return (long)(i / q_blk) * q_blk_stride + (long)s * q_seq + (long)(i % q_blk) * q_pos; }
    __device__ long k_row(int s, int r) const { return (long)s * k_seq + (long)r * k_pos; }
    __device__ float drop(int s, int head, int i, int r) const {
        if (p_drop <= 0.f) return 1.f;
        if (cross) {
            const long item_local = ((long)s * q_blk + i % q_blk) * heads + head;
            return drop_scale(seed, site, step + (uint32_t)(i / q_blk), (uint32_t)(item_local * nk + r), p_drop);
        }
        return drop_scale(seed, site, 0u, (uint32_t)((((long)s * heads + head) * idx_L + i) * idx_L + r), p_drop);
    }
    __device__ bool key_on(int s, int r) const { return key_mask == nullptr || key_mask[(long)s * ld_mask + r] != 0.f; }
    // keys [0, key_end) can be visible to the queries [q0, q0 + 32) of a tile
    __device__ int key_end(int q0) const {
        if (!causal) return nk;
        const int e = q0 + kTile < nq ? q0 + kTile : nq;
        return e < nk ? e : nk;
    }
};

// rows [row0, row0 + 32) of a head slice into shared memory [32][W]; rows past n are zero
__device__ __forceinline__ void stage_rows(float* __restrict__ dst, int W, int dk, int n_valid, const float* __restrict__ src, long ld, int head,
                                           const TiledAttn& a, int s, int i0, bool keys) {
#pragma unroll 4
    for (int e = threadIdx.x; e < kTile * dk; e += kThreads) {
        const int j = e / dk, c = e % dk;
        float x = 0.f;
        if (i0 + j < n_valid) x = src[(keys ? a.k_row(s, i0 + j) : a.q_row(s, i0 + j)) * ld + head * dk + c];
        dst[j * W + c] = x;
    }
}

template <int NC>
__global__ void __launch_bounds__(kThreads, 1) attn_tiled_forward_kernel(TiledAttn a, ActView out) {
    extern __shared__ __align__(16) float sm[];
    const int dk = a.dk, W = dk + 4, dk4 = dk >> 2;
    float* sK = sm;
    float* sV = sK + kTile * W;
    float* sQ = sV + kTile * W;
    const int s = blockIdx.x, head = blockIdx.y, q0 = a.q_lo + blockIdx.z * kTile;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    stage_rows(sQ, W, dk, a.nq, a.q, a.ld_q, head, a, s, q0, false);
    float m[kPerWarp], l[kPerWarp], acc[kPerWarp][NC];
#pragma unroll
    for (int u = 0; u < kPerWarp; ++u) {
        m[u] = -INFINITY; l[u] = 0.f;
#pragma unroll
        for (int i = 0; i < NC; ++i) acc[u][i] = 0.f;
    }
    const int k_end = a.key_end(q0);
    for (int k0 = 0; k0 < k_end; k0 += kTile) {
        __syncthreads();
        stage_rows(sK, W, dk, a.nk, a.k, a.ld_kv, head, a, s, k0, true);
        stage_rows(sV, W, dk, a.nk, a.v, a.ld_kv, head, a, s, k0, true);
        __syncthreads();
        const int r = k0 + lane;
        const bool key = r < a.nk && a.key_on(s, r);
#pragma unroll
        for (int u = 0; u < kPerWarp; ++u) {
            const int ql = warp * kPerWarp + u, qi = q0 + ql;
            if (qi >= a.nq) break;
            const bool on = key && (!a.causal || r <= qi);
            const float sc = on ? __fmul_rn(t_dot(sQ + ql * W, sK + lane * W, dk4), a.scale) : -INFINITY;
            const float m_new = fmaxf(m[u], t_wmax(sc));
            if (m_new == -INFINITY) continue;                   // every key so far masked: nothing to add
            const float corr = expf(m[u] - m_new);
            const float e = expf(sc - m_new);
            l[u] = l[u] * corr + t_wsum(e);
            m[u] = m_new;
            const float w = on ? e * a.drop(s, head, qi, r) : 0.f;
#pragma unroll
            for (int i = 0; i < NC; ++i) acc[u][i] *= corr;
            for (int j = 0; j < kTile; ++j) {
                const float wj = __shfl_sync(0xffffffffu, w, j);
#pragma unroll
                for (int i = 0; i < NC; ++i) {
                    const int c = lane + 32 * i;
                    if (c < dk) acc[u][i] = fmaf(wj, sV[j * W + c], acc[u][i]);
                }
            }
        }
    }
#pragma unroll
    for (int u = 0; u < kPerWarp; ++u) {
        const int qi = q0 + warp * kPerWarp + u;
        if (qi >= a.nq) break;
        const long row = a.q_row(s, qi);
        const float inv = 1.0f / l[u];
#pragma unroll
        for (int i = 0; i < NC; ++i) {
            const int c = lane + 32 * i;
            if (c >= dk) continue;
            const float x = acc[u][i] * inv;
            const long o = row * out.ld + head * dk + c;
            out.f[o] = x;
            if (out.hi != nullptr) split_f32(x, out.hi[o], out.lo[o]);
        }
    }
}

// Row pass: self-attention writes (max, 1 / sum, delta) of each query, cross-attention delta alone, into dq[row, head * dk + 0..2]
__global__ void __launch_bounds__(kThreads, 1) attn_tiled_rows_kernel(TiledAttn a) {
    extern __shared__ __align__(16) float sm[];
    const int dk = a.dk, W = dk + 4, dk4 = dk >> 2;
    float* sK = sm;
    float* sV = sK + kTile * W;
    float* sQ = sV + kTile * W;
    float* sD = sQ + kTile * W;
    const int s = blockIdx.x, head = blockIdx.y, q0 = blockIdx.z * kTile;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (!a.cross) stage_rows(sQ, W, dk, a.nq, a.q, a.ld_q, head, a, s, q0, false);
    stage_rows(sD, W, dk, a.nq, a.d_out, a.ld_do, head, a, s, q0, false);
    float m[kPerWarp], l[kPerWarp], d[kPerWarp];
#pragma unroll
    for (int u = 0; u < kPerWarp; ++u) { m[u] = -INFINITY; l[u] = 0.f; d[u] = 0.f; }
    const int k_end = a.key_end(q0);
    for (int k0 = 0; k0 < k_end; k0 += kTile) {
        __syncthreads();
        if (!a.cross) stage_rows(sK, W, dk, a.nk, a.k, a.ld_kv, head, a, s, k0, true);
        stage_rows(sV, W, dk, a.nk, a.v, a.ld_kv, head, a, s, k0, true);
        __syncthreads();
        const int r = k0 + lane;
#pragma unroll
        for (int u = 0; u < kPerWarp; ++u) {
            const int ql = warp * kPerWarp + u, qi = q0 + ql;
            if (qi >= a.nq) break;
            const float dov = r < a.nk ? __fmul_rn(t_dot(sD + ql * W, sV + lane * W, dk4), a.drop(s, head, qi, r)) : 0.f;
            if (a.cross) {
                const float p = r < a.nk ? a.probs[(a.q_row(s, qi) * a.heads + head) * a.nk + r] : 0.f;
                d[u] += t_wsum(p * dov);
                continue;
            }
            const bool on = r < a.nk && a.key_on(s, r) && (!a.causal || r <= qi);
            const float sc = on ? __fmul_rn(t_dot(sQ + ql * W, sK + lane * W, dk4), a.scale) : -INFINITY;
            const float m_new = fmaxf(m[u], t_wmax(sc));
            if (m_new == -INFINITY) continue;
            const float corr = expf(m[u] - m_new);
            const float e = expf(sc - m_new);
            l[u] = l[u] * corr + t_wsum(e);
            d[u] = d[u] * corr + t_wsum(e * dov);
            m[u] = m_new;
        }
    }
    if (lane != 0) return;
#pragma unroll
    for (int u = 0; u < kPerWarp; ++u) {
        const int qi = q0 + warp * kPerWarp + u;
        if (qi >= a.nq) break;
        float* st = a.dq + a.q_row(s, qi) * a.ld_dq + head * dk;
        if (a.cross) { st[0] = d[u]; continue; }
        const float inv = 1.0f / l[u];
        st[0] = m[u]; st[1] = inv; st[2] = d[u] * inv;
    }
}

// Scores and dO . V products are rounded (__fmul_rn, no FMA contraction) exactly as the row pass rounded them, so a query with a single
// visible key gets P = 1 and dS = 0 exactly.
// P_ir (probability before dropout) and dS_ir = P_ir (Z_ir dO_i . V_r - delta_i) * scale of query i (tile row qi of sQ / sD) against key r
// (tile row kr of sK / sV); st = (max, 1 / sum, delta) of query i, or delta alone (cross)
__device__ __forceinline__ void tiled_p_ds(const TiledAttn& a, int s, int head, int i, int r, const float* qv, const float* dov_row, const float* kv,
                                           const float* vv, const float* st, float& pz, float& ds) {
    pz = 0.f; ds = 0.f;
    if (i >= a.nq || r >= a.nk || (a.causal && r > i)) return;
    const int dk4 = a.dk >> 2;
    float p, delta;
    if (a.cross) {
        p = a.probs[(a.q_row(s, i) * a.heads + head) * a.nk + r];
        delta = st[0];
    } else {
        if (!a.key_on(s, r)) return;
        p = expf(__fmul_rn(t_dot(qv, kv, dk4), a.scale) - st[0]) * st[1];
        delta = st[2];
    }
    const float z = a.drop(s, head, i, r);
    pz = p * z;
    ds = p * (__fmul_rn(t_dot(dov_row, vv, dk4), z) - delta) * a.scale;
}

// dK / dV: one CTA per (sequence, head, tile of 32 keys); warp w owns keys w*4 .. w*4+3 of the tile, lane j = query j of each query tile
template <int NC>
__global__ void __launch_bounds__(kThreads, 1) attn_tiled_dkv_kernel(TiledAttn a, int accumulate) {
    extern __shared__ __align__(16) float sm[];
    const int dk = a.dk, W = dk + 4;
    float* sK = sm;
    float* sV = sK + kTile * W;
    float* sQ = sV + kTile * W;
    float* sD = sQ + kTile * W;
    float* sS = sD + kTile * W;             // [32][3] statistics of the query tile
    const int s = blockIdx.x, head = blockIdx.y, k0 = blockIdx.z * kTile;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (!a.cross) stage_rows(sK, W, dk, a.nk, a.k, a.ld_kv, head, a, s, k0, true);
    stage_rows(sV, W, dk, a.nk, a.v, a.ld_kv, head, a, s, k0, true);
    float gk[kPerWarp][NC], gv[kPerWarp][NC];
#pragma unroll
    for (int u = 0; u < kPerWarp; ++u)
#pragma unroll
        for (int i = 0; i < NC; ++i) { gk[u][i] = 0.f; gv[u][i] = 0.f; }
    for (int q0 = a.causal ? k0 : 0; q0 < a.nq; q0 += kTile) {          // causal: the query tiles before this key tile see none of its keys
        __syncthreads();
        stage_rows(sQ, W, dk, a.nq, a.q, a.ld_q, head, a, s, q0, false);
        stage_rows(sD, W, dk, a.nq, a.d_out, a.ld_do, head, a, s, q0, false);
        if (threadIdx.x < kTile * 3) {
            const int j = threadIdx.x / 3, c = threadIdx.x % 3;
            sS[threadIdx.x] = q0 + j < a.nq ? a.dq[a.q_row(s, q0 + j) * a.ld_dq + head * dk + c] : 0.f;
        }
        __syncthreads();
        const int i = q0 + lane;
#pragma unroll
        for (int u = 0; u < kPerWarp; ++u) {
            const int kl = warp * kPerWarp + u;
            if (k0 + kl >= a.nk) break;
            float pz, ds;
            tiled_p_ds(a, s, head, i, k0 + kl, sQ + lane * W, sD + lane * W, sK + kl * W, sV + kl * W, sS + lane * 3, pz, ds);
            for (int j = 0; j < kTile; ++j) {
                const float wv = __shfl_sync(0xffffffffu, pz, j), wk = __shfl_sync(0xffffffffu, ds, j);
#pragma unroll
                for (int c_ = 0; c_ < NC; ++c_) {
                    const int c = lane + 32 * c_;
                    if (c < dk) {
                        gv[u][c_] = fmaf(wv, sD[j * W + c], gv[u][c_]);
                        gk[u][c_] = fmaf(wk, sQ[j * W + c], gk[u][c_]);
                    }
                }
            }
        }
    }
#pragma unroll
    for (int u = 0; u < kPerWarp; ++u) {
        const int r = k0 + warp * kPerWarp + u;
        if (r >= a.nk) break;
        const long row = a.k_row(s, r) * a.ld_dkv + head * dk;
#pragma unroll
        for (int c_ = 0; c_ < NC; ++c_) {
            const int c = lane + 32 * c_;
            if (c >= dk) continue;
            a.dk_[row + c] = accumulate ? a.dk_[row + c] + gk[u][c_] : gk[u][c_];
            a.dv[row + c] = accumulate ? a.dv[row + c] + gv[u][c_] : gv[u][c_];
        }
    }
}

// dQ: one CTA per (sequence, head, tile of 32 queries); warp w owns queries w*4 .. w*4+3, lane r = key r of each key tile
template <int NC>
__global__ void __launch_bounds__(kThreads, 1) attn_tiled_dq_kernel(TiledAttn a) {
    extern __shared__ __align__(16) float sm[];
    const int dk = a.dk, W = dk + 4;
    float* sK = sm;
    float* sV = sK + kTile * W;
    float* sQ = sV + kTile * W;
    float* sD = sQ + kTile * W;
    float* sS = sD + kTile * W;
    const int s = blockIdx.x, head = blockIdx.y, q0 = blockIdx.z * kTile;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (!a.cross) stage_rows(sQ, W, dk, a.nq, a.q, a.ld_q, head, a, s, q0, false);
    stage_rows(sD, W, dk, a.nq, a.d_out, a.ld_do, head, a, s, q0, false);
    if (threadIdx.x < kTile * 3) {          // this tile's statistics, read before its dq rows are overwritten below
        const int j = threadIdx.x / 3, c = threadIdx.x % 3;
        sS[threadIdx.x] = q0 + j < a.nq ? a.dq[a.q_row(s, q0 + j) * a.ld_dq + head * dk + c] : 0.f;
    }
    float g[kPerWarp][NC];
#pragma unroll
    for (int u = 0; u < kPerWarp; ++u)
#pragma unroll
        for (int i = 0; i < NC; ++i) g[u][i] = 0.f;
    const int k_end = a.key_end(q0);
    for (int k0 = 0; k0 < k_end; k0 += kTile) {
        __syncthreads();
        stage_rows(sK, W, dk, a.nk, a.k, a.ld_kv, head, a, s, k0, true);
        stage_rows(sV, W, dk, a.nk, a.v, a.ld_kv, head, a, s, k0, true);
        __syncthreads();
#pragma unroll
        for (int u = 0; u < kPerWarp; ++u) {
            const int ql = warp * kPerWarp + u;
            if (q0 + ql >= a.nq) break;
            float pz, ds;
            tiled_p_ds(a, s, head, q0 + ql, k0 + lane, sQ + ql * W, sD + ql * W, sK + lane * W, sV + lane * W, sS + ql * 3, pz, ds);
            for (int j = 0; j < kTile; ++j) {
                const float w = __shfl_sync(0xffffffffu, ds, j);
#pragma unroll
                for (int c_ = 0; c_ < NC; ++c_) {
                    const int c = lane + 32 * c_;
                    if (c < dk) g[u][c_] = fmaf(w, sK[j * W + c], g[u][c_]);
                }
            }
        }
    }
#pragma unroll
    for (int u = 0; u < kPerWarp; ++u) {
        const int qi = q0 + warp * kPerWarp + u;
        if (qi >= a.nq) break;
        float* o = a.dq + a.q_row(s, qi) * a.ld_dq + head * dk;
#pragma unroll
        for (int c_ = 0; c_ < NC; ++c_) {
            const int c = lane + 32 * c_;
            if (c < dk) o[c] = g[u][c_];
        }
    }
}

// columns per lane of the accumulators: the smallest instantiated width that covers dk (dk <= 256)
inline int tiled_nc(int dk) { return dk <= 32 ? 1 : dk <= 64 ? 2 : dk <= 128 ? 4 : 8; }

// every footprint is at most 4 tiles x 32 rows x 260 floats + 96 (134 KB at dk 256): past the default 48 KB from dk 96 on
template <class K>
int set_smem(K kernel, std::atomic<unsigned long long>& configured) {
    if (first_use_on_device(configured)) CAPB_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    return 0;
}

size_t tiled_smem(int dk, int tiles) { return sizeof(float) * ((size_t)tiles * kTile * (dk + 4) + 3 * kTile); }

template <int NC>
int forward_nc(const TiledAttn& a, int seqs, ActView out, cudaStream_t st) {
    static std::atomic<unsigned long long> configured{0};
    const size_t smem = tiled_smem(a.dk, 3);
    if (set_smem(attn_tiled_forward_kernel<NC>, configured)) return 1;
    attn_tiled_forward_kernel<NC><<<dim3(seqs, a.heads, cdiv(a.nq - a.q_lo, kTile)), kThreads, smem, st>>>(a, out);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

template <int NC>
int backward_nc(const TiledAttn& a, int seqs, int accumulate, cudaStream_t st) {
    static std::atomic<unsigned long long> c_rows{0}, c_kv{0}, c_q{0};
    const size_t smem = tiled_smem(a.dk, 4);
    if (set_smem(attn_tiled_rows_kernel, c_rows) || set_smem(attn_tiled_dkv_kernel<NC>, c_kv) || set_smem(attn_tiled_dq_kernel<NC>, c_q))
        return 1;
    attn_tiled_rows_kernel<<<dim3(seqs, a.heads, cdiv(a.nq, kTile)), kThreads, smem, st>>>(a);
    CAPB_CHECK_CUDA(cudaGetLastError());
    attn_tiled_dkv_kernel<NC><<<dim3(seqs, a.heads, cdiv(a.nk, kTile)), kThreads, smem, st>>>(a, accumulate);
    CAPB_CHECK_CUDA(cudaGetLastError());
    attn_tiled_dq_kernel<NC><<<dim3(seqs, a.heads, cdiv(a.nq, kTile)), kThreads, smem, st>>>(a);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}

int check_shape(int dk, const char* what) {
    if ((dk & 3) != 0 || dk < 4 || dk > 256) {
        set_error(std::string(what) + " (key-tiled form): the head width must be a multiple of 4 between 4 and 256, got " + std::to_string(dk));
        return 1;
    }
    return 0;
}

// the dropout element index is 32-bit: refuse where it would wrap (the masks would repeat)
int check_index(long elements, float p, const char* what) {
    if (p > 0.f && elements >= (1l << 32)) {
        set_error(std::string(what) + ": " + std::to_string(elements) + " dropout elements per launch reach 2^32, where the 32-bit dropout index "
                  "wraps (DESIGN.md, 'Region counts')");
        return 1;
    }
    return 0;
}

TiledAttn self_args(int n_keys, int heads, int dk, int idx_L, long b_stride, long p_stride, const float* q, const float* k, const float* v, long ld,
                    const float* key_mask, long ld_mask, unsigned long long seed, int site, float p) {
    TiledAttn a{};
    a.nq = n_keys; a.nk = n_keys; a.dk = dk; a.heads = heads; a.q_blk = n_keys; a.q_blk_stride = 0;
    a.q_seq = b_stride; a.q_pos = p_stride; a.k_seq = b_stride; a.k_pos = p_stride;
    a.q = q; a.k = k; a.v = v; a.ld_q = ld; a.ld_kv = ld;
    a.scale = 1.0f / sqrtf((float)dk); a.p_drop = p; a.seed = seed; a.site = (uint32_t)site; a.step = 0; a.cross = 0; a.idx_L = idx_L;
    a.key_mask = key_mask; a.ld_mask = ld_mask;
    return a;
}

}  // namespace

int attn_tiled_forward_launch(int seqs, int n_keys, int heads, int dk, int idx_L, long b_stride, long p_stride, const float* q, const float* k, const float* v,
                              long ld, const float* key_mask, long ld_mask, unsigned long long seed, int site, float p, ActView out, cudaStream_t st, int causal,
                              int q_lo, int q_hi) {
    if (q_hi < 0) q_hi = n_keys;
    if (seqs <= 0 || n_keys <= 0 || q_hi <= q_lo) return 0;
    if (check_shape(dk, "self-attention") || check_index((long)seqs * heads * idx_L * idx_L, p, "self-attention")) return 1;
    CAPB_REQUIRE(q_lo >= 0 && (causal ? q_hi <= n_keys : (q_lo == 0 && q_hi == n_keys)),
                 "self-attention (key-tiled form): a query range needs the causal form, and stays within the keys");
    TiledAttn a = self_args(n_keys, heads, dk, idx_L, b_stride, p_stride, q, k, v, ld, key_mask, ld_mask, seed, site, p);
    a.nq = q_hi; a.q_lo = q_lo; a.causal = causal;
    switch (tiled_nc(dk)) {
        case 1: return forward_nc<1>(a, seqs, out, st);
        case 2: return forward_nc<2>(a, seqs, out, st);
        case 4: return forward_nc<4>(a, seqs, out, st);
        default: return forward_nc<8>(a, seqs, out, st);
    }
}

int attn_tiled_backward(const TiledAttn& a, int seqs, int accumulate, cudaStream_t st) {
    switch (tiled_nc(a.dk)) {
        case 1: return backward_nc<1>(a, seqs, accumulate, st);
        case 2: return backward_nc<2>(a, seqs, accumulate, st);
        case 4: return backward_nc<4>(a, seqs, accumulate, st);
        default: return backward_nc<8>(a, seqs, accumulate, st);
    }
}

int attn_tiled_self_backward_launch(int seqs, int n_keys, int heads, int dk, int idx_L, long b_stride, long p_stride, const float* q, const float* k,
                                    const float* v, long ld, unsigned long long seed, int site, float p, const float* d_out, long ld_do, float* dq, float* dk_,
                                    float* dv, long ld_d, const float* key_mask, long ld_mask, cudaStream_t st, int causal) {
    if (seqs <= 0 || n_keys <= 0) return 0;
    if (check_shape(dk, "self-attention backward") || check_index((long)seqs * heads * idx_L * idx_L, p, "self-attention backward")) return 1;
    CAPB_REQUIRE(dq != q && dq != k && dq != v && dq != d_out, "self-attention backward (key-tiled form): dq holds the row statistics, it must not alias an input");
    TiledAttn a = self_args(n_keys, heads, dk, idx_L, b_stride, p_stride, q, k, v, ld, key_mask, ld_mask, seed, site, p);
    a.causal = causal;
    a.d_out = d_out; a.ld_do = ld_do; a.dq = dq; a.dk_ = dk_; a.dv = dv; a.ld_dq = ld_d; a.ld_dkv = ld_d;
    return attn_tiled_backward(a, seqs, 0, st);
}

int attn_tiled_cross_backward_launch(int B, int rpi1, int n_steps, int row_mod, int heads, int dk, int R, const float* q, long ld_q, const float* kk,
                                     const float* vv, long ld_kv, unsigned long long seed, int site, int step, float p, const float* probs, const float* d_out,
                                     long ld_do, float* dq, long ld_dq, float* dkk, float* dvv, long ld_dkv, cudaStream_t st) {
    if (B <= 0 || rpi1 <= 0 || R <= 0) return 0;
    if (check_shape(dk, "decoder attention backward") || check_index((long)row_mod * heads * R, p, "decoder attention backward")) return 1;
    CAPB_REQUIRE(dq != q && dq != d_out && dq != kk && dq != vv, "decoder attention backward (key-tiled form): dq holds the row statistics, it must not alias an input");
    TiledAttn a{};
    a.nq = rpi1 * n_steps; a.nk = R; a.dk = dk; a.heads = heads; a.q_blk = rpi1; a.q_blk_stride = row_mod;
    a.q_seq = rpi1; a.q_pos = 1; a.k_seq = R; a.k_pos = 1;
    a.q = q; a.k = kk; a.v = vv; a.d_out = d_out; a.dq = dq; a.dk_ = dkk; a.dv = dvv;
    a.ld_q = ld_q; a.ld_kv = ld_kv; a.ld_do = ld_do; a.ld_dq = ld_dq; a.ld_dkv = ld_dkv;
    a.scale = 1.0f / sqrtf((float)dk); a.p_drop = p; a.seed = seed; a.site = (uint32_t)site; a.step = (uint32_t)step; a.cross = 1; a.idx_L = 0;
    a.probs = probs;
    return attn_tiled_backward(a, B, 1, st);
}

CAPB_DEFINE_SALT_SETTER(dropout_salt_set_attn)

}  // namespace capb200

using namespace capb200;

extern "C" {

int capb200_mha_forward(int form, int train, int B, int R, int heads, int dk, const float* q, const float* k, const float* v, long ld, const float* mask,
                        long ld_mask, unsigned long long seed, int site, float p, float* out, long ld_out, void* stream) {
    CAPB_REQUIRE(form >= 0 && form <= 2, "form is 0 (automatic), 1 (staged) or 2 (key-tiled)");
    CAPB_REQUIRE(B > 0 && R > 0 && heads > 0 && dk > 0 && q && k && v && out, "bad argument");
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (!train) {
        ActView o;
        o.f = out; o.ld = ld_out;
        return enc_self_attention_launch(B, R, heads, dk, q, k, v, ld, mask, ld_mask, o, st, form);
    }
    if (dropout_salt_set_all(0ull, st)) return 1;
    return seq_attn_train_launch(B, R, 0, R, heads, dk, 0, R, R, 1, q, k, v, ld, seed, site, p, out, ld_out, mask, ld_mask, st, form);
}

int capb200_mha_self_backward(int form, int B, int R, int heads, int dk, const float* q, const float* k, const float* v, long ld, const float* mask,
                              long ld_mask, unsigned long long seed, int site, float p, const float* d_out, long ld_do, float* dq, float* dk_, float* dv,
                              long ld_d, void* stream) {
    CAPB_REQUIRE(form >= 0 && form <= 2, "form is 0 (automatic), 1 (staged) or 2 (key-tiled)");
    CAPB_REQUIRE(B > 0 && R > 0 && heads > 0 && dk > 0 && q && k && v && d_out && dq && dk_ && dv, "bad argument");
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (dropout_salt_set_all(0ull, st)) return 1;
    return seq_attn_backward_launch(B, R, heads, dk, 0, R, R, 1, q, k, v, ld, seed, site, p, d_out, ld_do, dq, dk_, dv, ld_d, mask, ld_mask, st, form);
}

int capb200_mha_causal_forward(int form, int B, int T, int q_lo, int q_hi, int heads, int dk, const float* q, const float* k, const float* v, long ld,
                               const float* key_mask, long ld_mask, unsigned long long seed, int site, float p, float* out, long ld_out, void* stream) {
    CAPB_REQUIRE(form >= 0 && form <= 2, "form is 0 (automatic), 1 (staged) or 2 (key-tiled)");
    CAPB_REQUIRE(B > 0 && T > 0 && heads > 0 && dk > 0 && 0 <= q_lo && q_lo < q_hi && q_hi <= T && q && k && v && out, "bad argument");
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (dropout_salt_set_all(0ull, st)) return 1;
    return seq_attn_train_launch(B, q_hi, q_lo, q_hi, heads, dk, 1, T, T, 1, q, k, v, ld, seed, site, p, out, ld_out, key_mask, ld_mask, st, form);
}

int capb200_mha_causal_backward(int form, int B, int T, int heads, int dk, const float* q, const float* k, const float* v, long ld, const float* key_mask,
                                long ld_mask, unsigned long long seed, int site, float p, const float* d_out, long ld_do, float* dq, float* dk_, float* dv,
                                long ld_d, void* stream) {
    CAPB_REQUIRE(form >= 0 && form <= 2, "form is 0 (automatic), 1 (staged) or 2 (key-tiled)");
    CAPB_REQUIRE(B > 0 && T > 0 && heads > 0 && dk > 0 && q && k && v && d_out && dq && dk_ && dv, "bad argument");
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (dropout_salt_set_all(0ull, st)) return 1;
    return seq_attn_backward_launch(B, T, heads, dk, 1, T, T, 1, q, k, v, ld, seed, site, p, d_out, ld_do, dq, dk_, dv, ld_d, key_mask, ld_mask, st, form);
}

int capb200_mha_cross_backward(int form, int B, int rpi, int n_steps, int heads, int dk, int R, const float* q, long ld_q, const float* kk, const float* vv,
                               long ld_kv, unsigned long long seed, int site, int step, float p, const float* probs, const float* d_out, long ld_do, float* dq,
                               long ld_dq, float* dkk, float* dvv, long ld_dkv, void* stream) {
    CAPB_REQUIRE(form >= 0 && form <= 2, "form is 0 (automatic), 1 (staged) or 2 (key-tiled)");
    CAPB_REQUIRE(B > 0 && rpi > 0 && n_steps > 0 && R > 0 && heads > 0 && dk > 0 && q && kk && vv && probs && d_out && dq && dkk && dvv, "bad argument");
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (dropout_salt_set_all(0ull, st)) return 1;
    return cross_attn_backward_launch(B, rpi, heads, dk, R, q, ld_q, kk, vv, ld_kv, seed, site, step, p, probs, d_out, ld_do, dq, ld_dq, dkk, dvv, ld_dkv, st,
                                      n_steps, 0, form);
}

}  // extern "C"
