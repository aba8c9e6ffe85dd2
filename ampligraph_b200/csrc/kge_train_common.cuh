// kge_train_common.cuh -- device helpers shared by the training kernels (kge_train.cu: the general kernel;
// kge_train_res.cu / kge_train_rot.cu: the trilinear and RotatE fast paths; kge_train_bucket.cu: the replaced-row bucket
// sum): fp32-pair float4 arithmetic, the gradient scatter, warp reductions, the per-model score and gradient arithmetic,
// the corruption draw, and the per-positive loss + dL/dscore of the five reference losses; on the host, the launch they
// share and the trilinear row-shape dispatch.
#pragma once
#include <float.h>
#include <math.h>

#include <type_traits>

#include "kge_internal.h"

namespace kge {

// --------------------------------------------------------------------------
// float4 helpers
// --------------------------------------------------------------------------
__device__ __forceinline__ float4 f4zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }
__device__ __forceinline__ float4 f4ld(const float *p) { return *reinterpret_cast<const float4 *>(p); }
__device__ __forceinline__ void f4st(float *p, float4 v) { *reinterpret_cast<float4 *>(p) = v; }
// float4 arithmetic as two fp32 pairs (pk2 / fma2 / mul2 / add2 of kge_common.cuh)
__device__ __forceinline__ float4 f4from(f32x2_t lo, f32x2_t hi)
{
    float4 r;
    upk2(lo, r.x, r.y);
    upk2(hi, r.z, r.w);
    return r;
}
#define KGE_LO(v) pk2((v).x, (v).y)
#define KGE_HI(v) pk2((v).z, (v).w)
__device__ __forceinline__ float4 operator+(float4 a, float4 b) { return f4from(add2(KGE_LO(a), KGE_LO(b)), add2(KGE_HI(a), KGE_HI(b))); }
__device__ __forceinline__ float4 f4neg(float4 a) { return make_float4(-a.x, -a.y, -a.z, -a.w); }
__device__ __forceinline__ float4 operator-(float4 a, float4 b) { return a + f4neg(b); }
__device__ __forceinline__ float4 operator*(float4 a, float4 b) { return f4from(mul2(KGE_LO(a), KGE_LO(b)), mul2(KGE_HI(a), KGE_HI(b))); }
__device__ __forceinline__ float4 operator*(float a, float4 b)
{
    const f32x2_t aa = pk2(a, a);
    return f4from(mul2(aa, KGE_LO(b)), mul2(aa, KGE_HI(b)));
}
__device__ __forceinline__ float4 f4fma(float4 a, float4 b, float4 c)
{
    return f4from(fma2(KGE_LO(a), KGE_LO(b), KGE_LO(c)), fma2(KGE_HI(a), KGE_HI(b), KGE_HI(c)));
}
__device__ __forceinline__ float4 f4fma(float a, float4 b, float4 c)
{
    const f32x2_t aa = pk2(a, a);
    return f4from(fma2(aa, KGE_LO(b), KGE_LO(c)), fma2(aa, KGE_HI(b), KGE_HI(c)));
}
__device__ __forceinline__ float f4hsum(float4 a) { return (a.x + a.y) + (a.z + a.w); }
__device__ __forceinline__ float sgnf(float x) { return (x > 0.f) ? 1.f : ((x < 0.f) ? -1.f : 0.f); }  // TF abs grad
__device__ __forceinline__ float4 f4sgn(float4 a) { return make_float4(sgnf(a.x), sgnf(a.y), sgnf(a.z), sgnf(a.w)); }
__device__ __forceinline__ float f4abssum(float4 a) { return (fabsf(a.x) + fabsf(a.y)) + (fabsf(a.z) + fabsf(a.w)); }

// --------------------------------------------------------------------------
// gradient scatter: red.global.add.v4.f32 straight from registers into the gradient table.
// -DKGE_PROFILE_NOSCATTER builds a profiling variant that drops the scatter (how much of the kernel the atomics cost).
// The product never tests a run-time flag here: a branch around every RED was measured to cost several percent before
// the H100 port (not re-measured).
// --------------------------------------------------------------------------
__device__ __forceinline__ void red_add_v4(float *g, float4 v)
{
#ifdef KGE_PROFILE_NOSCATTER
    if (v.x != 1.2345e38f) return;  // profiling build: the scatter is dropped, v stays live
#endif
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(g), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
                 : "memory");
}
// The general kernel's form: a gradient row plus a float offset, added after v has been formed (writing row + off at the
// call site, before v, gives ptxas a different instruction order and changes the schedule of the general kernel).
__device__ __forceinline__ void red_add_v4(float *row, int off, float4 v) { red_add_v4(row + off, v); }

// RotatE's modulus and unit vector use the MUFU approximations (sqrt.approx: 2^-23 relative, rsqrt.approx: 2 ulp), far
// inside the 1e-4 training tolerance; the RANKING kernels keep the correctly rounded sqrt because their scores must be
// bit-identical to the oracle.
// single-instruction MUFU forms (flush-to-zero: a denormal x = re^2 + im^2 means a residual below 1e-19)
__device__ __forceinline__ float sqrt_approx(float x)
{
    float r;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ float rsqrt_approx(float x)
{
    float r;
    asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

__device__ __forceinline__ void warp_sum2(float &a, float &b)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
    }
}

// Two warp sums for the price of five shuffles (instead of ten): after the xor-16 step the lower half-warp carries a and
// the upper one b; four more steps finish each sum inside its half.  On return lanes [0,16) hold sum(a), lanes [16,32) sum(b).
__device__ __forceinline__ float warp_sum2t(float a, float b, int lane)
{
    const bool hi16 = (lane & 16) != 0;
    float k = hi16 ? b : a;
    k += __shfl_xor_sync(0xffffffffu, hi16 ? a : b, 16);
    k += __shfl_xor_sync(0xffffffffu, k, 8);
    k += __shfl_xor_sync(0xffffffffu, k, 4);
    k += __shfl_xor_sync(0xffffffffu, k, 2);
    k += __shfl_xor_sync(0xffffffffu, k, 1);
    return k;
}

// Four warp sums for the price of six shuffles: a transposed butterfly.  After the xor-16 step the lower half-warp
// carries v0, v1 and the upper one v2, v3; after the xor-8 step each quarter-warp carries ONE value; three more
// steps finish the sum inside the quarter.  On return lanes [8q, 8q+8) hold the full sum of value q.
__device__ __forceinline__ float warp_sum4t(float v0, float v1, float v2, float v3, int lane)
{
    const bool hi16 = (lane & 16) != 0, hi8 = (lane & 8) != 0;
    float k0 = hi16 ? v2 : v0, k1 = hi16 ? v3 : v1;
    k0 += __shfl_xor_sync(0xffffffffu, hi16 ? v0 : v2, 16);
    k1 += __shfl_xor_sync(0xffffffffu, hi16 ? v1 : v3, 16);
    float k = hi8 ? k1 : k0;
    k += __shfl_xor_sync(0xffffffffu, hi8 ? k0 : k1, 8);
    k += __shfl_xor_sync(0xffffffffu, k, 4);
    k += __shfl_xor_sync(0xffffffffu, k, 2);
    k += __shfl_xor_sync(0xffffffffu, k, 1);
    return k;
}

// --------------------------------------------------------------------------
// explicit shared-memory accessors (32-bit shared addresses) and register-pinning helpers of the fast paths
// (kge_train_res.cu, kge_train_rot.cu)
// --------------------------------------------------------------------------
__device__ __forceinline__ float4 lds4(uint32_t a)
{
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a));
    return v;
}
__device__ __forceinline__ float lds_f(uint32_t a)
{
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ int lds_i(uint32_t a)
{
    int v;
    asm volatile("ld.shared.s32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ void sts_f(uint32_t a, float v) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(a), "f"(v) : "memory"); }
__device__ __forceinline__ void sts_i(uint32_t a, int v) { asm volatile("st.shared.s32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ void mbar_init_s(uint32_t bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx_s(uint32_t bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait_s(uint32_t bar, uint32_t parity)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "RES_WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra RES_DONE;\n"
        "bra RES_WAIT_LOOP;\n"
        "RES_DONE:\n"
        "}\n" ::"r"(bar),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void bulk_load_s(uint32_t smem_dst, const void *gmem_src, uint32_t bytes, uint32_t bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_dst),
                 "l"(gmem_src), "r"(bytes), "r"(bar)
                 : "memory");
}
// The front end rematerialises cheap values (kernel parameters, %tid-derived addresses) inside the long per-positive
// loop instead of keeping them in registers -- a dozen ld.param / shift / mad per trip of the inner loops.  Passing a
// value through an empty asm makes it opaque: it is computed once and stays in its register.
#define KGE_KEEP32(x) asm volatile("" : "+r"(x))
#define KGE_KEEP64(x) asm volatile("" : "+l"(x))
#define KGE_KEEPF(x) asm volatile("" : "+f"(x))
__device__ __forceinline__ void red4(char *row, uint32_t byte_off, float4 v) { red_add_v4(reinterpret_cast<float *>(row + byte_off), v); }

// --------------------------------------------------------------------------
// Per-model arithmetic of the training kernels, one float4 chunk at a time.  The general kernel (kge_train.cu), the fast
// paths (kge_train_res.cu, kge_train_rot.cu) and the owner-computes gradient sum (kge_train_bucket.cu) all compute a
// model's scores and gradients with these functions, so their scores agree bit for bit and every g * Q term the bucket
// sum forms is the one the fused kernel would scatter.  A two-half (re / im) result is returned one half (H = 0: re,
// 1: im) at a time, so each half can be scattered as soon as it is formed (results returned through reference
// arguments were measured to change the fast paths' instruction schedule).
// --------------------------------------------------------------------------

// Query vectors of the trilinear models (DistMult: HALVES = 1; ComplEx / HolE: HALVES = 2): the score of a corruption
// is <row, Q>, and its replaced row's gradient is g * Q.  Subject replaced: Q0(p, o); object replaced: Q1(s, p).
template <int HALVES, int H>
__device__ __forceinline__ float4 query_subj(float4 pr, float4 pi, float4 orr, float4 oi)
{
    if constexpr (HALVES == 1) return pr * orr;
    else if constexpr (H == 0) return f4fma(pi, oi, pr * orr);
    else return pr * oi - pi * orr;
}
template <int HALVES, int H>
__device__ __forceinline__ float4 query_obj(float4 sr, float4 si, float4 pr, float4 pi)
{
    if constexpr (HALVES == 1) return sr * pr;
    else if constexpr (H == 0) return sr * pr - si * pi;
    else return f4fma(sr, pi, si * pr);
}
// both halves at once, for the bucket sum (with HALVES = 1, qi is not written)
template <int HALVES>
__device__ __forceinline__ void query_subj(float4 pr, float4 pi, float4 orr, float4 oi, float4 &qr, float4 &qi)
{
    qr = query_subj<HALVES, 0>(pr, pi, orr, oi);
    if constexpr (HALVES == 2) qi = query_subj<HALVES, 1>(pr, pi, orr, oi);
}
template <int HALVES>
__device__ __forceinline__ void query_obj(float4 sr, float4 si, float4 pr, float4 pi, float4 &qr, float4 &qi)
{
    qr = query_obj<HALVES, 0>(sr, si, pr, pi);
    if constexpr (HALVES == 2) qi = query_obj<HALVES, 1>(sr, si, pr, pi);
}
// Gradient rows of a trilinear positive's kept rows.  U is everything that sat in the subject slot (gP s + the
// subject-replaced corruptions' sum_j g_j r_j), X everything in the object slot, W1 the object-replaced share of X.
// Entity rows: d/ds f(s,p,X) = Q0(p, X), d/do f(U,p,o) = Q1(U, p).  Relation row: d/dp [f(U,p,o) + f(s,p,W1)].
template <int HALVES, int H>
__device__ __forceinline__ float4 trilinear_grad_p(float4 sr, float4 si, float4 orr, float4 oi, float4 Ur, float4 Ui,
                                                   float4 W1r, float4 W1i)
{
    if constexpr (HALVES == 1) return f4fma(Ur, orr, sr * W1r);
    else if constexpr (H == 0) return f4fma(Ur, orr, Ui * oi) + f4fma(sr, W1r, si * W1i);
    else return (Ur * oi - Ui * orr) + (sr * W1i - si * W1r);
}

// RotatE (RotatE.py:76-104), relation row = rotation table row [cos(phi) | sin(phi)] = (c, sn), f = -sum_d |R(phi) s - o|.
// With (a, b) = g * residual / |residual|: df/do = (a, b); df/ds = -R(-phi)(a, b); df/dphi = a y_im - b y_re, y = R(phi) s.
// FP32-issue bound: every float4 operation is four fp32 instructions (negations are FADD / FFMA operand modifiers).
// sum of the four moduli of (re, im): x = re^2 + im^2, one MUFU.SQRT each
__device__ __forceinline__ float rot_modsum(float4 re, float4 im)
{
    const float4 x = f4fma(im, im, re * re);
    return (sqrt_approx(x.x) + sqrt_approx(x.y)) + (sqrt_approx(x.z) + sqrt_approx(x.w));
}
// (a, b) = g * (re, im) / |(re, im)|: one MUFU.RSQ on max(x, FLT_MIN), the smallest x whose rsqrt.approx.ftz is finite,
// so every normal x gets its own rsqrt and an exactly-zero residual gives 0 * 2^63 = 0 (the reference's gradient is NaN
// there); below FLT_MIN the result is g * (re, im) * 2^63, at most |g| per component
__device__ __forceinline__ void rot_unit(float4 re, float4 im, float g, float4 &a, float4 &b)
{
    const float4 x = f4fma(im, im, re * re);
    const float4 inv = g * make_float4(rsqrt_approx(fmaxf(x.x, FLT_MIN)), rsqrt_approx(fmaxf(x.y, FLT_MIN)),
                                       rsqrt_approx(fmaxf(x.z, FLT_MIN)), rsqrt_approx(fmaxf(x.w, FLT_MIN)));
    a = re * inv;
    b = im * inv;
}
// R(phi)(rr, ri) = (rr c - ri sn, rr sn + ri c)
template <int H>
__device__ __forceinline__ float4 rot_rotate(float4 rr, float4 ri, float4 c, float4 sn)
{
    if constexpr (H == 0) return f4fma(f4neg(ri), sn, rr * c);
    else return f4fma(rr, sn, ri * c);
}
// the residual of a replaced subject, R(phi) r - o, as two dependent fmas per component
template <int H>
__device__ __forceinline__ float4 rot_residual_subj(float4 rr, float4 ri, float4 c, float4 sn, float4 orr, float4 oi)
{
    if constexpr (H == 0) return f4fma(f4neg(ri), sn, f4fma(rr, c, f4neg(orr)));
    else return f4fma(ri, c, f4fma(rr, sn, f4neg(oi)));
}
// -R(-phi)(a, b) = (-(a c + b sn), a sn - b c): the subject-side gradient of a residual whose unit vector is (a, b)
template <int H>
__device__ __forceinline__ float4 rot_back(float4 a, float4 b, float4 c, float4 sn)
{
    if constexpr (H == 0) return f4fma(f4neg(b), sn, f4neg(a) * c);
    else return f4fma(f4neg(b), c, a * sn);
}
// acc + a y_im - b y_re: the dphi accumulation
__device__ __forceinline__ float4 rot_dphi(float4 a, float4 b, float4 yr, float4 yi, float4 acc)
{
    return f4fma(f4neg(b), yr, f4fma(a, yi, acc));
}

// Corruption r = j*B + i of the step (the reference's tile order): the injected negatives when the caller supplied
// them, else the Philox draw.  keep = 1: the subject is kept and the object replaced by repl.
__device__ __forceinline__ void corruption_of(const TrainParams &p, unsigned long long r, int &keep, int &repl)
{
    if (p.neg_ent) { repl = p.neg_ent[r]; keep = p.neg_keep[r] ? 1 : 0; }
    else draw_corruption(p.seed, p.step, r, p.n_ent, &keep, &repl);
}

// --------------------------------------------------------------------------
// Dynamic assignment of positives to warps.  A static stride (warp w takes w, w + n_warps, ...) quantises the launch to
// ceil(B / n_warps) rounds -- cfg2: 27,212 positives over 1,776 warps = 15.3, so a third of the warps run a 16th round
// while the rest idle (4 %); cfg4: 9.1 -> 10 rounds (9 %).  Instead every warp starts on its own index and draws the
// following ones from a counter: the draw for the NEXT positive is issued before the current one is processed, so its
// latency is never seen.  The counters reset themselves: the last warp to retire (all draws are complete by then)
// zeroes both words, so consecutive launches on one stream need no memset and the scheme survives graph replay.
// --------------------------------------------------------------------------
// (a FLOAT counter on purpose: the compiler -- nvcc for atomicAdd(), ptxas for atom.add / atom.inc in inline PTX, u32 and u64,
// even with a laundered addend -- aggregates a warp's integer atomic adds (VOTE + POPC, one ATOMG) and reads the result back
// with a shuffle right after it, which puts the whole L2 round trip, microseconds when HBM is saturated, at the top of every
// positive: measured markedly slower on an HBM-resident table before the H100 port.  atom.add.f32 is left alone;
// counts are exact below 2^24, the host falls back to the static stride for larger batches.)
#define KGE_SCHED_MAX_B (1ll << 24)
__device__ __forceinline__ float sched_draw(unsigned *sched)  // the caller converts when it consumes the value, not here
{
    float v;
    asm volatile("atom.relaxed.gpu.global.add.f32 %0, [%1], 0f3F800000;" : "=f"(v) : "l"(sched) : "memory");
    return v;
}
__device__ __forceinline__ void sched_retire(unsigned *sched, long long n_warps, int lane)
{
    if (sched && lane == 0) {
        const unsigned d = atomicAdd(sched + 1, 1u);
        if ((long long)d == n_warps - 1) { sched[0] = 0u; sched[1] = 0u; }
    }
}

// --------------------------------------------------------------------------
// per-positive loss and dL/dscore (warp-cooperative; lanes stride over j).
// in: P, sc[j] = N_j.  out: sc[j] = dL/dN_j, returns loss_i, *dP.
// --------------------------------------------------------------------------
// x / y for y in a range where the IEEE slow path (denormal operands) cannot matter: reciprocal + multiply, no FCHK branch
#ifdef KGE_FAST_LOSS_MATH
__device__ __forceinline__ float fdiv(float x, float y) { return __fdividef(x, y); }
#else
__device__ __forceinline__ float fdiv(float x, float y) { return x / y; }
#endif
__device__ __forceinline__ float log_sigmoid(float x) { return fminf(x, 0.f) - log1pf(expf(-fabsf(x))); }
__device__ __forceinline__ float sigmoidf(float x) { return fdiv(1.f, 1.f + expf(-x)); }
#define KGE_CLIP_LO (-75.0f)  // loss_functions.py:32
#define KGE_CLIP_HI (75.0f)   // loss_functions.py:35

static __device__ __forceinline__ float loss_and_dscores(const TrainParams &p, float P, float *sc, int lane, float *dP_out)
{
    const int eta = p.eta;
    const float w = (p.reduction == KGE_REDUCE_MEAN) ? 1.f / (float)eta : 1.f;
    float loss = 0.f, dP = 0.f;
    switch (p.loss) {
    case KGE_LOSS_PAIRWISE: {  // loss_functions.py:305-307
        float acc = 0.f, ds = 0.f;
        for (int j = lane; j < eta; j += 32) {
            float x = p.margin - P + sc[j];
            float d = (x >= 0.f) ? w : 0.f;  // TF maximum(): tie goes to the first argument
            acc += fmaxf(x, 0.f);
            ds += d;
            sc[j] = d;
        }
        loss = w * warp_sum(acc);
        dP = -warp_sum(ds);
        break;
    }
    case KGE_LOSS_NLL: {  // loss_functions.py:376-382 (positive term counted eta times)
        const float w2 = (p.reduction == KGE_REDUCE_MEAN) ? 1.f / (2.f * (float)eta) : 1.f;
        float Pc = fminf(fmaxf(P, KGE_CLIP_LO), KGE_CLIP_HI);
        float inP = (P >= KGE_CLIP_LO && P <= KGE_CLIP_HI) ? 1.f : 0.f;
        float acc = 0.f;
        for (int j = lane; j < eta; j += 32) {
            float N = sc[j];
            float Nc = fminf(fmaxf(N, KGE_CLIP_LO), KGE_CLIP_HI);
            float inN = (N >= KGE_CLIP_LO && N <= KGE_CLIP_HI) ? 1.f : 0.f;
            float e = expf(Nc);
            acc += logf(1.f + e);
            sc[j] = w2 * inN * (e / (1.f + e));
        }
        float ep = expf(-Pc);
        loss = w2 * ((float)eta * logf(1.f + ep) + warp_sum(acc));
        dP = -w2 * (float)eta * inP * (ep / (1.f + ep));
        break;
    }
    case KGE_LOSS_ABSOLUTE_MARGIN: {  // loss_functions.py:461-463
        float acc = 0.f;
        for (int j = lane; j < eta; j += 32) {
            float x = p.margin + sc[j];
            acc += fmaxf(x, 0.f);
            sc[j] = (x >= 0.f) ? w : 0.f;
        }
        loss = w * warp_sum(acc) - w * (float)eta * P;
        dP = -w * (float)eta;
        break;
    }
    case KGE_LOSS_SELF_ADVERSARIAL: {  // loss_functions.py:563-572, softmax NOT detached
        // with x = -N - margin, t = exp(-|x|):  log_sigmoid(x) = min(x,0) - log1p(t) and
        // sigmoid(N + margin) = sigmoid(-x) = (x < 0 ? 1 : t) / (1 + t): one exp + one log1p per corruption
        if (eta <= 32) {  // one corruption per lane: everything stays in registers
            const bool on = lane < eta;
            const float N = on ? sc[lane] : 0.f;
            const float mx = warp_max(on ? p.alpha * N : -INFINITY);
            const float e = on ? expf(p.alpha * N - mx) : 0.f;
            const float x = -N - p.margin, t = expf(-fabsf(x));
            const float lj = fminf(x, 0.f) - log1pf(t);
            const float sg = fdiv((x < 0.f) ? 1.f : t, 1.f + t);
            float z = e, sl = e * lj;
            warp_sum2(z, sl);
            const float S = fdiv(sl, z), pj = fdiv(e, z);
            if (on) sc[lane] = w * (pj * sg - p.alpha * pj * (lj - S));
            loss = -log_sigmoid(p.margin + P) - w * S;
            dP = -sigmoidf(-(p.margin + P));
            break;
        }
        float mx = -INFINITY;
        for (int j = lane; j < eta; j += 32) mx = fmaxf(mx, p.alpha * sc[j]);
        mx = warp_max(mx);
        float z = 0.f, sl = 0.f;
        for (int j = lane; j < eta; j += 32) {
            float e = expf(p.alpha * sc[j] - mx);
            z += e;
            sl += e * log_sigmoid(-sc[j] - p.margin);
        }
        z = warp_sum(z);
        float S = warp_sum(sl) / z;
        for (int j = lane; j < eta; j += 32) {
            float N = sc[j];
            float pj = expf(p.alpha * N - mx) / z;
            float lj = log_sigmoid(-N - p.margin);
            sc[j] = w * (pj * sigmoidf(N + p.margin) - p.alpha * pj * (lj - S));
        }
        loss = -log_sigmoid(p.margin + P) - w * S;
        dP = -sigmoidf(-(p.margin + P));
        break;
    }
    case KGE_LOSS_MULTICLASS_NLL: {  // loss_functions.py:647-653
        float Pc = fminf(fmaxf(P, KGE_CLIP_LO), KGE_CLIP_HI);
        float inP = (P >= KGE_CLIP_LO && P <= KGE_CLIP_HI) ? 1.f : 0.f;
        float acc = 0.f;
        for (int j = lane; j < eta; j += 32) acc += expf(fminf(fmaxf(sc[j], KGE_CLIP_LO), KGE_CLIP_HI));
        float pe = expf(Pc);
        float D = w * warp_sum(acc) + pe;
        for (int j = lane; j < eta; j += 32) {
            float N = sc[j];
            float inN = (N >= KGE_CLIP_LO && N <= KGE_CLIP_HI) ? 1.f : 0.f;
            sc[j] = w * inN * expf(fminf(fmaxf(N, KGE_CLIP_LO), KGE_CLIP_HI)) / D;
        }
        loss = -logf(pe / D);
        dP = inP * (pe / D - 1.f);
        break;
    }
    }
    *dP_out = dP;
    return loss;
}

// Host side of every training launcher: slot.warps warps per CTA, each with its slot of shared memory, on as many CTAs as
// are co-resident (each strides over the positives) but no more than the positives need.
template <class Kernel>
static cudaError_t launch_persistent(Kernel kern, const TrainParams &p, const TrainSlot &slot, int sm_count, cudaStream_t st)
{
    if (p.B == 0) return cudaSuccess;
    const int threads = slot.warps * 32;
    const size_t smem = (size_t)slot.warps * slot.region_bytes;
    cudaError_t e = allow_dynamic_smem(kern, smem);
    if (e != cudaSuccess) return e;
    int occ = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, threads, smem);
    if (e != cudaSuccess) return e;
    if (occ < 1) return cudaErrorLaunchOutOfResources;
    const long long want = (p.B + slot.warps - 1) / slot.warps, cap = (long long)occ * sm_count;
    kern<<<(int)(want < cap ? want : cap), threads, smem, st>>>(p);
    return cudaGetLastError();
}

// Host side of the trilinear fast paths: returns launch(std::integral_constant<int, HALVES>, std::integral_constant<int,
// NIT>) for the row shape of model and nit.  HALVES = 1 for DistMult, 2 (re / im) for ComplEx and HolE; NIT is the number
// of float4 chunks per lane and half.  NIT = 4 (rows of 512+ floats per half) is DistMult's alone: only its per-lane state
// fits the register file (kge_create).
template <class Launch>
static cudaError_t dispatch_trilinear_shape(int model, int nit, Launch &&launch)
{
    using one = std::integral_constant<int, 1>;
    using two = std::integral_constant<int, 2>;
    const bool halves2 = model != KGE_DISTMULT;
    if (nit <= 1) return halves2 ? launch(two{}, one{}) : launch(one{}, one{});
    if (nit == 2) return halves2 ? launch(two{}, two{}) : launch(one{}, two{});
    if (halves2) return cudaErrorInvalidValue;
    return launch(one{}, std::integral_constant<int, 4>{});
}

}  // namespace kge
