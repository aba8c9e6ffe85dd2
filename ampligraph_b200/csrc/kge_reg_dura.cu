// kge_reg_dura.cu -- the DURA regulariser of a step's positives (Zhang, Cai and Wang, "Duality-Induced Regularizer for
// Tensor Factorization Based Knowledge Graph Completion", NeurIPS 2020), sm_90a.
//
// L_DURA = sum_b sum_d [ w_n (m_h + m_t) + w_p m_r (m_h + m_t) ] over the B positives (h_b, r_b, t_b) of a step, where
// m_x = |x_d|^2: x[d]^2 for the one-half layouts, x[d]^2 + x[kp + d]^2 for the two-half ones.  Its gradient is, component
// by component on each half,
//   d/dh_d = 2 (w_n + w_p m_r) h_d,   d/dt_d = 2 (w_n + w_p m_r) t_d,   d/dr_d = 2 w_p (m_h + m_t) r_d.
// An entity row's gradient needs the sum of m_r over its occurrences and a relation row's the sum of m_h + m_t over its
// own, so N3's one-writer-per-row form (a count times a function of the row) does not apply.  kge_dura_kernel runs one
// thread per (positive, float4 chunk of a half), like the 1vsAll chain pass: it reads its chunk of h, r and t and adds the
// three gradient chunks with red.global.add.v4.f32.  The gradient is the same fp32 sum in any order, but the order is the
// REDs' arrival order, so it is bit-for-bit repeatable only where every partial sum is exact.  Each thread's loss terms
// are summed in fp64 across the warp, then added with one fp64 atomic per warp.  With w_p = 0 the relation row is neither
// read nor written.  Padding columns hold 0, so their gradient is 0.  DESIGN.md 3.16.
#include "kge_train_common.cuh"

namespace kge {

#define DURA_THREADS 256

// m = |z|^2 of one component (explicit roundings: no contraction)
template <int HALVES>
__device__ __forceinline__ float dura_sq(float re, float im)
{
    return HALVES == 2 ? __fadd_rn(__fmul_rn(re, re), __fmul_rn(im, im)) : __fmul_rn(re, re);
}

// One component of a positive: a = w_n + w_p m_r and s = m_h + m_t; adds 2a h, 2a t and 2 w_p s r to the gradient chunks
// and returns the loss term s a.
template <int HALVES>
__device__ __forceinline__ float dura_component(const DuraParams &p, float hr, float hi, float rr, float ri, float tr,
                                                float ti, float &ghr, float &ghi, float &grr, float &gri, float &gtr,
                                                float &gti)
{
    const float s = __fadd_rn(dura_sq<HALVES>(hr, hi), dura_sq<HALVES>(tr, ti));
    const float a = __fadd_rn(p.w_norm, __fmul_rn(p.w_prod, dura_sq<HALVES>(rr, ri)));
    const float ce = __fmul_rn(2.f, a), cr = __fmul_rn(p.w_prod2, s);
    ghr = __fmul_rn(ce, hr);
    gtr = __fmul_rn(ce, tr);
    grr = __fmul_rn(cr, rr);
    if (HALVES == 2) {
        ghi = __fmul_rn(ce, hi);
        gti = __fmul_rn(ce, ti);
        gri = __fmul_rn(cr, ri);
    }
    return __fmul_rn(s, a);
}

template <int HALVES>
__global__ void __launch_bounds__(DURA_THREADS) kge_dura_kernel(const DuraParams p)
{
    const int nq4 = p.kp / 4;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    double loss = 0.0;
    if (idx < p.B * nq4) {
        const long long b = idx / nq4;
        const int d = (int)(idx - b * nq4) * 4, di = HALVES == 2 ? p.kp + d : d;
        const int hi_ = p.triples[3 * b], ri_ = p.triples[3 * b + 1], ti_ = p.triples[3 * b + 2];
        const bool prod = p.w_prod > 0.f;
        const float *hrow = p.ent + (size_t)hi_ * p.ld, *trow = p.ent + (size_t)ti_ * p.ld;
        const float4 hr = f4ld(hrow + d), hm = HALVES == 2 ? f4ld(hrow + di) : f4zero();
        const float4 tr = f4ld(trow + d), tm = HALVES == 2 ? f4ld(trow + di) : f4zero();
        float4 rr = f4zero(), rm = f4zero();
        if (prod) {
            const float *rrow = p.rel + (size_t)ri_ * p.ld;
            rr = f4ld(rrow + d);
            if (HALVES == 2) rm = f4ld(rrow + di);
        }
        float4 ghr, ghm = f4zero(), grr, grm = f4zero(), gtr, gtm = f4zero();
        loss += (double)dura_component<HALVES>(p, hr.x, hm.x, rr.x, rm.x, tr.x, tm.x, ghr.x, ghm.x, grr.x, grm.x, gtr.x, gtm.x);
        loss += (double)dura_component<HALVES>(p, hr.y, hm.y, rr.y, rm.y, tr.y, tm.y, ghr.y, ghm.y, grr.y, grm.y, gtr.y, gtm.y);
        loss += (double)dura_component<HALVES>(p, hr.z, hm.z, rr.z, rm.z, tr.z, tm.z, ghr.z, ghm.z, grr.z, grm.z, gtr.z, gtm.z);
        loss += (double)dura_component<HALVES>(p, hr.w, hm.w, rr.w, rm.w, tr.w, tm.w, ghr.w, ghm.w, grr.w, grm.w, gtr.w, gtm.w);
        float *gh = p.grad_ent + (size_t)hi_ * p.ld, *gt = p.grad_ent + (size_t)ti_ * p.ld;
        red_add_v4(gh + d, ghr);
        red_add_v4(gt + d, gtr);
        if (HALVES == 2) {
            red_add_v4(gh + di, ghm);
            red_add_v4(gt + di, gtm);
        }
        if (prod) {
            float *gr = p.grad_rel + (size_t)ri_ * p.ld;
            red_add_v4(gr + d, grr);
            if (HALVES == 2) red_add_v4(gr + di, grm);
        }
        if (d == 0 && p.stamp_ent) {
            p.stamp_ent[hi_] = p.stamp;
            p.stamp_ent[ti_] = p.stamp;
            if (prod && p.stamp_rel) p.stamp_rel[ri_] = p.stamp;
        }
    }
    // fp64 across the warp: the terms of the exactly representable tables then sum without rounding
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) loss += __shfl_xor_sync(0xffffffffu, loss, o);
    if ((threadIdx.x & 31) == 0 && p.loss && loss != 0.0) atomicAdd(p.loss, loss);
}

cudaError_t launch_dura(const DuraParams &p, int halves, cudaStream_t st)
{
    if (p.B == 0) return cudaSuccess;
    const unsigned grid = (unsigned)((p.B * (p.kp / 4) + DURA_THREADS - 1) / DURA_THREADS);
    return dispatch_value<1, 2>(halves, [&](auto H) {
        kge_dura_kernel<decltype(H)::value><<<grid, DURA_THREADS, 0, st>>>(p);
        return cudaGetLastError();
    });
}

}  // namespace kge
