// net6.cuh -- constants of the latent grid, the fp32 head tables the tensor-core kernels read, and the canonical fused
// softmax-expectation + inverse scalar transform (lzero/policy/scaling_transform.py:82-92) shared by every kernel that turns
// categorical logits into a scalar (k_net_tc, mlp.cu, ez.cu, k_inverse_scalar).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace lz {

constexpr int kC = 64;          // latent channels (num_channels)
constexpr int kHW = 6;          // latent height == width
constexpr int kP = kHW * kHW;   // 36 pixels

struct Head {                   // fp32 tables of conv1x1 -> BN -> ReLU -> Linear(hc*P->hid) -> BN1d -> ReLU -> Linear(hid->K)
    const float *s2, *t2;       // [hid]  BN1d folded, Linear bias folded into t2
    const float *b2;            // [K]    bias of the last Linear
    int hc, hid, K;             // hid == 0: no FC part on the tensor cores (EfficientZero's reward head, ez.cu)
};

// torch.sign(v) * (((sqrt(1 + 4 eps (|v| + 1 + eps)) - 1) / (2 eps))^2 - 1), eps = 0.001, evaluated
// in fp32 in the operation order of scaling_transform.py:89-91.
__device__ __forceinline__ float inverse_scalar_transform(float v)
{
    const float eps = 0.001f;
    float t = __fadd_rn(__fadd_rn(fabsf(v), 1.0f), eps);
    t = __fadd_rn(1.0f, __fmul_rn(__fmul_rn(4.0f, eps), t));
    t = __fdiv_rn(__fsub_rn(__fsqrt_rn(t), 1.0f), __fmul_rn(2.0f, eps));
    float o = __fsub_rn(__fmul_rn(t, t), 1.0f);
    float sg = (v > 0.0f) ? 1.0f : ((v < 0.0f) ? -1.0f : 0.0f);
    return __fmul_rn(sg, o);
}

__device__ __forceinline__ float warp_sum(float v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// softmax(logits) . support  ->  inverse transform  (scaling_transform.py:82-92).
//
// ONE canonical evaluation order for every kernel of the library (so that the fused search, the step-wise drive and the stand-alone
// lz_inverse_scalar_transform agree bit for bit): the K logits are dealt to 128 virtual threads (k mod 128), each folds its logits
// in increasing k into a running (max m, sum s of exp(x - m), sum w of exp(x - m) * support_k); the 128 triples are combined as
// 4 groups of 32 (xor-shuffle max, maximum of the 4 group maxima in group order, rescale by exp(m - M), xor-shuffle sums, the 4
// group sums added in group order).  k_net_tc's FC2 stage runs it natively (thread = output k, heads_fc in net_tc.cu); a single
// warp emulates it here with 4 virtual threads per lane.
__device__ __forceinline__ void softmax_push(float &m, float &s, float &w, float x, float sup)
{
    // one exponential per logit, no divergent branch: t = exp(-|x - m|) is the rescale factor of the old sums when x is the new
    // maximum and the new term otherwise (exp(-inf) = 0 for the first logit)
    const float t = __expf(-fabsf(x - m));      // ex2.approx: ~2 ulp; the terms that matter have |x - m| of a few units
    const bool gt = x > m;
    s = gt ? fmaf(s, t, 1.0f) : s + t;
    w = gt ? fmaf(w, t, sup) : fmaf(t, sup, w);
    m = gt ? x : m;
}
__device__ __forceinline__ float support_at(float support_min, float support_step, int k) { return fmaf(support_step, (float)k, support_min); }

__device__ __forceinline__ float categorical_to_scalar(const float *logits /*shared or global*/, int K,
                                                       float support_min, float support_step, int lane)
{
    float m[4], s[4], w[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) { m[j] = -INFINITY; s[j] = 0.0f; w[j] = 0.0f; }
    for (int k0 = 0; k0 < K; k0 += 128) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int k = k0 + j * 32 + lane;
            if (k < K) softmax_push(m[j], s[j], w[j], logits[k], support_at(support_min, support_step, k));
        }
    }
    float M = warp_max(m[0]);
#pragma unroll
    for (int j = 1; j < 4; ++j) M = fmaxf(M, warp_max(m[j]));
    float S = 0.0f, W = 0.0f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float sc = (m[j] == -INFINITY) ? 0.0f : expf(m[j] - M);
        S += warp_sum(s[j] * sc);
        W += warp_sum(w[j] * sc);
    }
    return inverse_scalar_transform(W / S);
}

}  // namespace lz
