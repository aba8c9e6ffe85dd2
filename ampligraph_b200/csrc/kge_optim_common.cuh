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

// d/dx lam*|x|^p = sign(x)*(lam*p*|x|^(p-1)): returns the second factor; *loss += lam*|x|^p, as one fma
__device__ __forceinline__ float lp_scale(float ax, int p, float lam, float *loss)
{
    const float pm1 = (p == 2) ? ax : (p == 3) ? __fmul_rn(ax, ax) : (p == 1) ? 1.f : powf(ax, (float)(p - 1));
    *loss = fmaf(__fmul_rn(pm1, ax), lam, *loss);
    return lam * (float)p * pm1;
}
// The regulariser's gradient sign(x)*s1, plus sign(x)*s2 in one fma for a second term; sign(+-0) = sign(NaN) = 0.
// Needs r.p > 0: the kernels instantiate REG only for a table that has a regulariser (the exchange kernel, which takes
// two tables, chooses per element).
__device__ __forceinline__ float reg_grad(float x, const RegParams &r, float *loss)
{
    const float ax = fabsf(x), sg = (x > 0.f) ? 1.f : ((x < 0.f) ? -1.f : 0.f);
    float g = __fmul_rn(sg, lp_scale(ax, r.p, r.lambda, loss));
    if (r.p2 > 0) g = fmaf(sg, lp_scale(ax, r.p2, r.lambda2, loss), g);
    return g;
}

// Which of the two slot buffers a kind reads and writes (kge_b200.h documents what each holds).  SGD's slot 0 exists
// only with momentum, RMSprop's slot 1 only when centered (mg) or with momentum (mom); every other use is fixed by the
// kind.  Every kernel and the host's argument check ask this one function.
__host__ __device__ __forceinline__ constexpr bool uses_slot0(int kind, float momentum)
{
    return kind != KGE_OPT_SGD || momentum != 0.f;
}
__host__ __device__ __forceinline__ constexpr bool uses_slot1(int kind, float momentum, int centered)
{
    return kind == KGE_OPT_ADAM || kind == KGE_OPT_ADADELTA || kind == KGE_OPT_ADAMAX || kind == KGE_OPT_NADAM ||
           kind == KGE_OPT_FTRL || (kind == KGE_OPT_RMSPROP && (centered != 0 || momentum != 0.f));
}

// One element of the legacy update rules (optimizers.py:255-291 -> tf.keras.optimizers.legacy.* and the training ops
// they call).  g is the summed gradient plus the regulariser's, a / b are slot 0 / slot 1.  Every operation is spelled
// out: fma is one rounding (fmaf), every other +, -, * rounds to fp32 on its own -- every product that feeds a sum is
// __fmul_rn, so that the compiler cannot contract it into an fma; a product that feeds / or sqrt cannot be contracted --
// / and sqrt are IEEE round-to-nearest (no fast-math), and 1-b1, 1-b2, 1-rho are fp32 subtractions.
// tests/optim_exact_oracle.py restates this order bit for bit:
//   SGD       momentum 0: x = fma(-g, lr, x);  else a = fma(a, mu, -(g*lr)), x = x + a
//   Adam      a = fma(g - a, 1-b1, a); b = fma(fma(g, g, -b), 1-b2, b); x -= (a*lr_t) / (sqrt(b) + eps)
//             lr_t = lr*sqrt(1-b2^t)/(1-b1^t), fp64 on the host, rounded once
//   Adagrad   a = fma(g, g, a); x -= (lr*g) / (sqrt(a) + eps)
//   RMSprop   momentum 0: a = fma(rho, a, (1-rho)*(g*g)); d = a, or when centered b = fma(rho, b, (1-rho)*g),
//             d = fma(-b, b, a); x -= (lr*g) / (sqrt(d) + eps)
//             momentum mu > 0 (ApplyRMSProp, never centered): a = fma(g*g - a, 1-rho, a);
//             b = fma(mu, b, (lr*g) / sqrt(a + eps)); x -= b
//   Adadelta  a = fma(rho, a, (1-rho)*(g*g)); u = (sqrt(b + eps) / sqrt(a + eps)) * g; x = fma(-lr, u, x);
//             b = fma(rho, b, (1-rho)*(u*u))
//   Adamax    a = fma(g - a, 1-b1, a); b = fmaxf(b2*b, |g|) (a NaN g is dropped, as fmaxf does);
//             x = fma(-lr_t, a / (b + eps), x);  lr_t = lr/(1-b1^t), fp64 on the host, rounded once
// Nadam and Ftrl round every operation on its own (no fma), as TensorFlow's separate ops (Nadam) and its CPU ApplyFtrl
// expression evaluate them; q holds their per-step scalars (kge_api.cu, optim_step):
//   Nadam     a = b1*a + (1-b1)*g; b = b2*b + (1-b2)*(g*g);
//             mb = (1-m_t)*(g / (1-s_new)) + m_t1*(a / (1-s_next)); x -= (lr*mb) / (sqrt(b / v_den) + eps)
//             row-decay mode, a row not looked up this step: a = b1*a, b = b2*b, x unchanged (nadam_decay)
//   Ftrl      gs = g, or g + shrinkx2*x when l2_shrinkage > 0 (ApplyFtrlV2); n1 = a + g*g;
//             P(y) = sqrt(y) when lr_power = -0.5, else powf(y, -lr_power);
//             b += gs - ((P(n1) - P(a)) / lr)*x; x = |b| > l1 ? (sign(b)*l1 - b) / (P(n1)/lr + l2x2) : 0; a = n1
template <int KIND>
__device__ __forceinline__ void apply_rule(float &x, float gg, float &a, float &b, const OptimParams &o,
                                           const OptimStep &q)
{
    if (KIND == KGE_OPT_ADAM) {
        a = fmaf(gg - a, 1.f - o.beta1, a);          // m += (g-m)(1-b1)
        b = fmaf(fmaf(gg, gg, -b), 1.f - o.beta2, b);  // v += (g^2-v)(1-b2)
        x -= (a * o.lr_t) / (sqrtf(b) + o.eps);
    } else if (KIND == KGE_OPT_ADAGRAD) {
        a = fmaf(gg, gg, a);
        x -= o.lr * gg / (sqrtf(a) + o.eps);
    } else if (KIND == KGE_OPT_RMSPROP) {
        const float g2 = __fmul_rn(gg, gg), step = __fmul_rn(o.lr, gg);
        if (o.momentum != 0.f) {
            a = fmaf(__fsub_rn(g2, a), 1.f - o.rho, a);
            b = fmaf(o.momentum, b, step / sqrtf(a + o.eps));
            x -= b;
        } else {
            a = fmaf(o.rho, a, __fmul_rn(1.f - o.rho, g2));
            float d = a;
            if (o.centered) {
                b = fmaf(o.rho, b, __fmul_rn(1.f - o.rho, gg));
                d = fmaf(-b, b, a);
            }
            x -= step / (sqrtf(d) + o.eps);
        }
    } else if (KIND == KGE_OPT_ADADELTA) {
        a = fmaf(o.rho, a, __fmul_rn(1.f - o.rho, __fmul_rn(gg, gg)));
        const float u = __fmul_rn(sqrtf(b + o.eps) / sqrtf(a + o.eps), gg);
        x = fmaf(-o.lr, u, x);
        b = fmaf(o.rho, b, __fmul_rn(1.f - o.rho, __fmul_rn(u, u)));
    } else if (KIND == KGE_OPT_ADAMAX) {
        a = fmaf(gg - a, 1.f - o.beta1, a);
        b = fmaxf(__fmul_rn(o.beta2, b), fabsf(gg));
        x = fmaf(-o.lr_t, a / (b + o.eps), x);
    } else if (KIND == KGE_OPT_NADAM) {
        a = __fadd_rn(__fmul_rn(o.beta1, a), __fmul_rn(1.f - o.beta1, gg));
        b = __fadd_rn(__fmul_rn(o.beta2, b), __fmul_rn(1.f - o.beta2, __fmul_rn(gg, gg)));
        const float mb = __fadd_rn(__fmul_rn(q.one_m_mt, gg / q.one_m_snew), __fmul_rn(q.m_t1, a / q.one_m_snext));
        x = __fsub_rn(x, __fmul_rn(o.lr, mb) / __fadd_rn(sqrtf(b / q.v_den), o.eps));
    } else if (KIND == KGE_OPT_FTRL) {
        const float gs = q.shrinkx2 > 0.f ? __fadd_rn(gg, __fmul_rn(q.shrinkx2, x)) : gg;
        const float n1 = __fadd_rn(a, __fmul_rn(gg, gg));
        const bool half = q.lr_power == -0.5f;
        const float p1 = half ? sqrtf(n1) : powf(n1, -q.lr_power), p0 = half ? sqrtf(a) : powf(a, -q.lr_power);
        b = __fadd_rn(b, __fsub_rn(gs, __fmul_rn(__fsub_rn(p1, p0) / o.lr, x)));
        const float den = __fadd_rn(p1 / o.lr, q.l2x2);
        x = fabsf(b) > q.l1 ? __fsub_rn(copysignf(q.l1, b), b) / den : 0.f;
        a = n1;
    } else {  // SGD (momentum optional)
        if (o.momentum != 0.f) { a = fmaf(a, o.momentum, -__fmul_rn(gg, o.lr)); x += a; }
        else x = fmaf(-gg, o.lr, x);
    }
}

template <int KIND, bool REG>
__device__ __forceinline__ float4 update4(float4 x4, float4 g4, float4 &a4, float4 &b4, const OptimParams &o,
                                          const OptimStep &q, const RegParams &reg, float &racc)
{
    float x[4] = {x4.x, x4.y, x4.z, x4.w}, g[4] = {g4.x, g4.y, g4.z, g4.w};
    float a[4] = {a4.x, a4.y, a4.z, a4.w}, b[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        float gg = g[e];
        if (REG) gg += reg_grad(x[e], reg, &racc);
        apply_rule<KIND>(x[e], gg, a[e], b[e], o, q);
    }
    a4 = make_float4(a[0], a[1], a[2], a[3]);
    b4 = make_float4(b[0], b[1], b[2], b[3]);
    return make_float4(x[0], x[1], x[2], x[3]);
}

// Nadam's row-decay mode on a row that was not looked up: m *= b1, v *= b2
__device__ __forceinline__ void nadam_decay4(float4 &a4, float4 &b4, const OptimParams &o)
{
    a4 = make_float4(__fmul_rn(o.beta1, a4.x), __fmul_rn(o.beta1, a4.y), __fmul_rn(o.beta1, a4.z), __fmul_rn(o.beta1, a4.w));
    b4 = make_float4(__fmul_rn(o.beta2, b4.x), __fmul_rn(o.beta2, b4.y), __fmul_rn(o.beta2, b4.z), __fmul_rn(o.beta2, b4.w));
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
    return dispatch_value<KGE_OPT_SGD, KGE_OPT_ADAM, KGE_OPT_ADAGRAD, KGE_OPT_RMSPROP, KGE_OPT_ADADELTA, KGE_OPT_ADAMAX,
                          KGE_OPT_NADAM, KGE_OPT_FTRL>(
        kind, [&](auto k) { return reg ? launch(k, std::true_type{}) : launch(k, std::false_type{}); });
}

}  // namespace kge
