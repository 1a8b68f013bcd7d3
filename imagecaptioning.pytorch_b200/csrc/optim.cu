// Fused gradient clamp + Adam update over a table of parameter tensors (C ABI capb200_adam_step in include/capb200.h).
//
// Reference: tools/train.py:193-196 -- utils.clip_gradient(optimizer, opt.grad_clip_value) (captioning/utils/misc.py:156-160: every
// param.grad clamped to [-c, c] in place) followed by optimizer.step() with torch.optim.Adam built by build_optimizer (misc.py:186-205).
// The stock path is ~125 launches and ~10 passes over the 85 M parameters of AoANet; here it is ONE launch and one pass: g, p, m, v read once, p, m, v (and the clamped g) written once.
// Arithmetic follows torch's single-tensor Adam term by term (lerp for exp_avg, mul + addcmul for exp_avg_sq, sqrt / bias2_sqrt + eps,
// addcdiv with -lr / bias1), so the result matches torch.optim.Adam to fp32 rounding (tests/test_gpu_ops.py).
#include "../../include/capb200.h"
#include "common.cuh"

namespace capb200 {

namespace {

constexpr int kChunk = 8192;        // elements per CTA (256 threads x 8 float4)

struct AdamScalars {
    float lr_over_bias1, bias2_sqrt, beta1, beta2, omb1, omb2, eps, weight_decay, clip;      // omb = 1 - beta, rounded from double like torch's python scalars
    int write_clamped;
};

__device__ __forceinline__ void adam_one(float& p, float& g, float& m, float& v, const AdamScalars& s) {
    if (s.clip > 0.f) g = fminf(fmaxf(g, -s.clip), s.clip);
    float gg = g;
    if (s.weight_decay != 0.f) gg = fmaf(s.weight_decay, p, gg);
    m = m + (gg - m) * s.omb1;                                // exp_avg.lerp_(grad, 1 - beta1)
    v = v * s.beta2 + s.omb2 * gg * gg;                       // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value = 1 - beta2)
    const float denom = sqrtf(v) / s.bias2_sqrt + s.eps;
    p = p - s.lr_over_bias1 * (m / denom);                     // param.addcdiv_(exp_avg, denom, value = -lr / bias1)
}

// table[i] = {p, g, m, v} (device pointers), numel[i]; chunks[c] = {tensor index, first element}
__global__ void __launch_bounds__(256) adam_kernel(const unsigned long long* __restrict__ table, const long long* __restrict__ numel,
                                                   const int2* __restrict__ chunks, AdamScalars s) {
    const int2 ch = chunks[blockIdx.x];
    const unsigned long long* row = table + 4l * ch.x;
    float* p = reinterpret_cast<float*>(row[0]);
    float* g = reinterpret_cast<float*>(row[1]);
    float* m = reinterpret_cast<float*>(row[2]);
    float* v = reinterpret_cast<float*>(row[3]);
    const long n = numel[ch.x];
    const long lo = (long)ch.y * kChunk;
    const long hi = (lo + kChunk < n) ? lo + kChunk : n;
    const bool vec = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) | reinterpret_cast<uintptr_t>(v)) & 15) == 0;
    if (vec) {
        const long hi4 = lo + ((hi - lo) & ~3l);
        for (long i = lo + 4l * threadIdx.x; i < hi4; i += 1024) {
            float4 P = *reinterpret_cast<float4*>(p + i), Gv = *reinterpret_cast<float4*>(g + i), M = *reinterpret_cast<float4*>(m + i),
                   V = *reinterpret_cast<float4*>(v + i);
            adam_one(P.x, Gv.x, M.x, V.x, s); adam_one(P.y, Gv.y, M.y, V.y, s); adam_one(P.z, Gv.z, M.z, V.z, s); adam_one(P.w, Gv.w, M.w, V.w, s);
            *reinterpret_cast<float4*>(p + i) = P; *reinterpret_cast<float4*>(m + i) = M; *reinterpret_cast<float4*>(v + i) = V;
            if (s.write_clamped) *reinterpret_cast<float4*>(g + i) = Gv;
        }
        for (long i = hi4 + threadIdx.x; i < hi; i += 256) {
            float P = p[i], Gs = g[i], M = m[i], V = v[i];
            adam_one(P, Gs, M, V, s);
            p[i] = P; m[i] = M; v[i] = V;
            if (s.write_clamped) g[i] = Gs;
        }
    } else {
        for (long i = lo + threadIdx.x; i < hi; i += 256) {
            float P = p[i], Gs = g[i], M = m[i], V = v[i];
            adam_one(P, Gs, M, V, s);
            p[i] = P; m[i] = M; v[i] = V;
            if (s.write_clamped) g[i] = Gs;
        }
    }
}

}  // namespace

}  // namespace capb200

using namespace capb200;

extern "C" int capb200_adam_chunk_elems(void) { return kChunk; }

extern "C" int capb200_adam_step(const unsigned long long* table, const long long* numel, const int* chunks, int n_chunks, double lr, double beta1,
                                 double beta2, double eps, double weight_decay, long step, double clip_value, int write_clamped, void* stream) {
    CAPB_REQUIRE(table != nullptr && numel != nullptr && chunks != nullptr && n_chunks >= 0, "null argument");
    CAPB_REQUIRE(step >= 1 && beta1 >= 0.0 && beta1 < 1.0 && beta2 >= 0.0 && beta2 < 1.0 && eps >= 0.0, "bad Adam hyper-parameters");
    if (n_chunks == 0) return 0;
    AdamScalars s;
    // the scalars are python floats (doubles) in torch's Adam and reach its kernels rounded once to fp32: same here
    const double bias1 = 1.0 - pow(beta1, (double)step);
    const double bias2 = 1.0 - pow(beta2, (double)step);
    s.lr_over_bias1 = (float)(lr / bias1);
    s.bias2_sqrt = (float)sqrt(bias2);
    s.beta1 = (float)beta1; s.beta2 = (float)beta2; s.omb1 = (float)(1.0 - beta1); s.omb2 = (float)(1.0 - beta2); s.eps = (float)eps;
    s.weight_decay = (float)weight_decay; s.clip = (float)clip_value; s.write_clamped = write_clamped;
    adam_kernel<<<n_chunks, 256, 0, static_cast<cudaStream_t>(stream)>>>(table, numel, reinterpret_cast<const int2*>(chunks), s);
    CAPB_CHECK_CUDA(cudaGetLastError());
    return 0;
}
