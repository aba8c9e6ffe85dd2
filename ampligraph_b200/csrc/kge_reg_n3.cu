// kge_reg_n3.cu -- the N3 regulariser of a step's positives (Lacroix, Usunier and Obozinski, ICML 2018, eq. 6), sm_90a.
//
// L_N3 = lambda_ent * sum_b sum_d (|s_bd|^3 + |o_bd|^3) + lambda_rel * sum_b sum_d |p_bd|^3 over the B positives of a
// step, where |z_d| is |x[d]| for the one-half layouts and the modulus of (x[d], x[kp + d]) for the two-half ones.  It is
// written per row: L_N3 = sum_rows lambda * c_row * sum_d |z_d|^3, c_row the row's occurrences as s or o (entity rows)
// or as p (relation rows), so every row has one writer:
//   1. kge_n3_count_kernel: one thread per positive, integer atomics into cnt[n_ent + n_rel] (order independent, so the
//      counts are deterministic).  The caller zeroes cnt first.
//   2. kge_n3_apply_kernel: one warp per row of the [ent | rel] block, grid stride; rows with c = 0 return at once.  The
//      warp forms m_d = |z_d| and adds c * 3 lambda * m_d * z_d to the row's gradient with a plain load-add-store (this
//      pass is the row's only writer while it runs, so the gradient is bit-for-bit repeatable), and adds
//      lambda * c * sum_d m_d^3 of its rows to the loss with one fp64 atomic per warp.
// Padding columns hold 0, so their m and gradient are 0.  DESIGN.md 3.15.
#include "kge_internal.h"

namespace kge {

#define N3_THREADS 256

// p.lambda_* == 0 tables are neither counted nor touched (their table and gradient pointers may be null)
__global__ void __launch_bounds__(N3_THREADS) kge_n3_count_kernel(const N3Params p)
{
    for (long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x; b < p.B; b += (long long)gridDim.x * blockDim.x) {
        const int32_t *t = p.triples + 3 * b;
        if (p.lambda_ent > 0.f) {
            atomicAdd(p.cnt + t[0], 1);
            atomicAdd(p.cnt + t[2], 1);
        }
        if (p.lambda_rel > 0.f) atomicAdd(p.cnt + p.n_ent + t[1], 1);
    }
}

// m = |z| of one component: the modulus of (re, im) for two halves (explicit roundings: no contraction), |re| for one
template <int HALVES>
__device__ __forceinline__ float n3_mod(float re, float im)
{
    return HALVES == 2 ? __fsqrt_rn(__fadd_rn(__fmul_rn(re, re), __fmul_rn(im, im))) : fabsf(re);
}

// sum += m^3; g += coef * m * z (component-wise)
template <int HALVES>
__device__ __forceinline__ void n3_component(float re, float im, float coef, float &g_re, float &g_im, float &sum)
{
    const float m = n3_mod<HALVES>(re, im), k = __fmul_rn(coef, m);
    sum = __fadd_rn(sum, __fmul_rn(__fmul_rn(m, m), m));
    g_re = __fadd_rn(g_re, __fmul_rn(k, re));
    if (HALVES == 2) g_im = __fadd_rn(g_im, __fmul_rn(k, im));
}

template <int HALVES>
__global__ void __launch_bounds__(N3_THREADS) kge_n3_apply_kernel(const N3Params p)
{
    const int lane = threadIdx.x & 31, nch = p.kp / 4;
    const long long warps = (long long)gridDim.x * (N3_THREADS / 32);
    double loss = 0.0;
    for (long long r = p.row_begin + (long long)blockIdx.x * (N3_THREADS / 32) + (threadIdx.x >> 5); r < p.row_end; r += warps) {
        const int c = p.cnt[r];
        if (c == 0) continue;
        const bool ent = r < p.n_ent;
        const long long row = ent ? r : r - p.n_ent;
        const float lam = ent ? p.lambda_ent : p.lambda_rel;
        const float coef = __fmul_rn(ent ? p.lambda3_ent : p.lambda3_rel, (float)c);  // c * 3 lambda
        const float4 *x = reinterpret_cast<const float4 *>((ent ? p.ent : p.rel) + row * p.ld);
        float4 *g = reinterpret_cast<float4 *>((ent ? p.grad_ent : p.grad_rel) + row * p.ld);
        float sum = 0.f;
        for (int ch = lane; ch < nch; ch += 32) {
            const float4 re = x[ch], im = HALVES == 2 ? x[nch + ch] : make_float4(0.f, 0.f, 0.f, 0.f);
            float4 gr = g[ch], gi = HALVES == 2 ? g[nch + ch] : make_float4(0.f, 0.f, 0.f, 0.f);
            n3_component<HALVES>(re.x, im.x, coef, gr.x, gi.x, sum);
            n3_component<HALVES>(re.y, im.y, coef, gr.y, gi.y, sum);
            n3_component<HALVES>(re.z, im.z, coef, gr.z, gi.z, sum);
            n3_component<HALVES>(re.w, im.w, coef, gr.w, gi.w, sum);
            g[ch] = gr;
            if (HALVES == 2) g[nch + ch] = gi;
        }
        sum = warp_sum(sum);
        loss += (double)lam * (double)c * (double)sum;
        if (lane == 0) {
            int *stamp = ent ? p.stamp_ent : p.stamp_rel;
            if (stamp) stamp[row] = p.stamp;
        }
    }
    if (lane == 0 && p.loss && loss != 0.0) atomicAdd(p.loss, loss);
}

cudaError_t launch_n3(const N3Params &p, int halves, int sm_count, cudaStream_t st)
{
    if (p.B == 0) return cudaSuccess;
    cudaError_t e = cudaMemsetAsync(p.cnt, 0, sizeof(int) * (size_t)(p.n_ent + p.n_rel), st);
    if (e != cudaSuccess) return e;
    const long long count_blocks = (p.B + N3_THREADS - 1) / N3_THREADS;
    kge_n3_count_kernel<<<(int)(count_blocks < 4096 ? count_blocks : 4096), N3_THREADS, 0, st>>>(p);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    // one warp per row, grid stride: at most 8 CTAs of 8 warps per SM (a full SM), fewer when there are few rows
    const long long rows = p.row_end - p.row_begin, need = (rows + N3_THREADS / 32 - 1) / (N3_THREADS / 32);
    const long long cap = 8ll * sm_count, blocks = need < cap ? need : cap;
    if (blocks == 0) return cudaSuccess;
    return dispatch_value<1, 2>(halves, [&](auto H) {
        kge_n3_apply_kernel<decltype(H)::value><<<(int)blocks, N3_THREADS, 0, st>>>(p);
        return cudaGetLastError();
    });
}

}  // namespace kge
