// kge_optim_common.cuh -- the per-element optimizer update and regulariser (sm_90a), shared by the dense, lazy,
// sharded and exchange kernels of kge_optim.cu and by the owner-per-row kernel of kge_train_bucket.cu, so that every
// path applies the same fp32 arithmetic; on the host, their launchers' choice of instantiation.
//
// Replaces OptimizerWrapper.minimize -> tf.keras.optimizers.legacy.*.apply_gradients (optimizers.py:136-168) and the
// regularisers attached to the tables (regularizers.py:14-37, EmbeddingLookupLayer.py:131-155).  The regulariser's
// gradient and loss are taken at the PRE-update value of each element.
#pragma once
#include <math.h>

#include <type_traits>

#include "kge_internal.h"

namespace kge {

// d/dx lam*|x|^p = lam*p*|x|^(p-1)*sign(x); *loss += lam*|x|^p
__device__ __forceinline__ float lp_term(float x, int p, float lam, float *loss)
{
    const float ax = fabsf(x), sg = (x > 0.f) ? 1.f : ((x < 0.f) ? -1.f : 0.f);
    const float pm1 = (p == 2) ? ax : (p == 3) ? ax * ax : (p == 1) ? 1.f : powf(ax, (float)(p - 1));
    *loss += lam * (pm1 * ax);
    return lam * (float)p * pm1 * sg;
}
__device__ __forceinline__ float reg_grad(float x, const RegParams &r, float *loss)
{
    float g = lp_term(x, r.p, r.lambda, loss);
    if (r.p2 > 0) g += lp_term(x, r.p2, r.lambda2, loss);
    return g;
}

// one element of the legacy update rules (optimizers.py:255-291 -> tf.keras.optimizers.legacy.*)
template <int KIND>
__device__ __forceinline__ void apply_rule(float &x, float gg, float &a, float &b, const OptimParams &o)
{
    if (KIND == KGE_OPT_ADAM) {
        a = fmaf(gg - a, 1.f - o.beta1, a);       // m += (g-m)(1-b1)
        b = fmaf(gg * gg - b, 1.f - o.beta2, b);  // v += (g^2-v)(1-b2)
        x -= (a * o.lr_t) / (sqrtf(b) + o.eps);
    } else if (KIND == KGE_OPT_ADAGRAD) {
        a = fmaf(gg, gg, a);
        x -= o.lr * gg / (sqrtf(a) + o.eps);
    } else {  // SGD (momentum optional)
        if (o.momentum != 0.f) { a = o.momentum * a - o.lr * gg; x += a; }
        else x -= o.lr * gg;
    }
}

template <int KIND, bool REG>
__device__ __forceinline__ float4 update4(float4 x4, float4 g4, float4 &a4, float4 &b4, const OptimParams &o,
                                          const RegParams &reg, float &racc)
{
    float x[4] = {x4.x, x4.y, x4.z, x4.w}, g[4] = {g4.x, g4.y, g4.z, g4.w};
    float a[4] = {a4.x, a4.y, a4.z, a4.w}, b[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        float gg = g[e];
        if (REG) gg += reg_grad(x[e], reg, &racc);
        apply_rule<KIND>(x[e], gg, a[e], b[e], o);
    }
    a4 = make_float4(a[0], a[1], a[2], a[3]);
    b4 = make_float4(b[0], b[1], b[2], b[3]);
    return make_float4(x[0], x[1], x[2], x[3]);
}

// block-reduce the per-thread regulariser loss and add it to the double accumulator
__device__ __forceinline__ void flush_reg_loss(float racc, double *reg_loss)
{
    racc = warp_sum(racc);
    __shared__ float part[32];
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = racc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < (int)((blockDim.x + 31) >> 5); ++w) t += (double)part[w];
        if (t != 0.0) atomicAdd(reg_loss, t);
    }
}

// Host side of every optimizer launcher: returns launch(std::integral_constant<int, KIND>, std::integral_constant<bool,
// REG>) for the optimizer kind and whether a regulariser is set, or cudaErrorInvalidValue for an unknown kind.
template <class Launch>
static cudaError_t dispatch_optimizer(int kind, bool reg, Launch &&launch)
{
    auto with_reg = [&](auto k) { return reg ? launch(k, std::true_type{}) : launch(k, std::false_type{}); };
    switch (kind) {
    case KGE_OPT_SGD: return with_reg(std::integral_constant<int, KGE_OPT_SGD>{});
    case KGE_OPT_ADAM: return with_reg(std::integral_constant<int, KGE_OPT_ADAM>{});
    case KGE_OPT_ADAGRAD: return with_reg(std::integral_constant<int, KGE_OPT_ADAGRAD>{});
    default: return cudaErrorInvalidValue;
    }
}

}  // namespace kge
