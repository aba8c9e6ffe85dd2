// kge_dropout.cu -- embedding dropout of the all-candidate steps (kge_one_vs_all_step, kge_one_vs_all_relation_step,
// kge_k_vs_all_step while kge_set_embedding_dropout is set; DESIGN.md 3.19).
//
// Inverted dropout of every embedding element a side's scores read: x~ = fp32(x * scale) where kept, +0 where dropped,
// scale = fp32(1 / (1 - p)).  The masks come from Philox4x32-10 (SideDropout in kge_internal.h), so nothing is stored:
//   prepare  writes the side's dropped candidate table into the workspace once (the five passes read it as s.cand),
//            zeroes the candidates' gradient buffer (the dX pass adds into it as s.grad_cand) and forms the query
//            vectors from the dropped query rows (each occurrence b of a row its own mask);
//   finish   adds fp32(scale * g~) of each kept candidate element to the raw gradient table (the candidate's gradient
//            summed over the batch first, then masked), and runs the chain pass of kge_train_1vsall.cu on the dropped
//            query rows, each occurrence's gradient masked by its own mask before it is added.
// The passes between them are the unchanged kernels of kge_train_1vsall.cu.
#include "kge_train_common.cuh"

namespace kge {

__device__ __forceinline__ u32x4 dropout_words(const SideDropout &d, long long row, int c, int tag)
{
    return philox4x32_10((uint32_t)row, (uint32_t)(c >> 2) | ((0x80u | (uint32_t)tag) << 24), (uint32_t)d.step,
                         (uint32_t)(d.step >> 32), (uint32_t)d.seed, (uint32_t)(d.seed >> 32));
}

// the mask of the 4 elements c .. c + 3 (c a multiple of 4) as 0 / 1 lanes
struct Keep4 {
    bool x, y, z, w;
};
__device__ __forceinline__ Keep4 dropout_keep4(const SideDropout &d, long long row, int c, int tag, uint32_t t)
{
    const u32x4 v = dropout_words(d, row, c, tag);
    return Keep4{(v.x >> 8) >= t, (v.y >> 8) >= t, (v.z >> 8) >= t, (v.w >> 8) >= t};
}
// fp32(v * scale) where kept, +0 where dropped: the dropped copy of a row chunk, and the raw gradient of a chunk
// from the gradient of its dropped copy
__device__ __forceinline__ float4 dropout_apply4(Keep4 k, float4 v, float scale)
{
    return make_float4(k.x ? __fmul_rn(v.x, scale) : 0.f, k.y ? __fmul_rn(v.y, scale) : 0.f,
                       k.z ? __fmul_rn(v.z, scale) : 0.f, k.w ? __fmul_rn(v.w, scale) : 0.f);
}

__host__ __device__ __forceinline__ int dropout_tag(int side, int role) { return 4 * (side + 1) + role; }  // side 1 = s, 2 = o, 3 = p

// out[r] = dropped copy of x[r] (ADD = false), or grad[r] += raw gradient of g[r] (ADD = true); one thread per float4
template <bool ADD>
__global__ void __launch_bounds__(256) kge_dropout_rows_kernel(const float *__restrict__ x, float *__restrict__ out,
                                                               long long rows, int ld, const SideDropout d, int tag,
                                                               uint32_t t, float scale)
{
    const int n4 = ld / 4;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= rows * n4) return;
    const long long r = idx / n4;
    const int c = (int)(idx - r * n4) * 4;
    const size_t off = (size_t)idx * 4;
    const float4 v = dropout_apply4(dropout_keep4(d, r, c, tag, t), f4ld(x + off), scale);
    f4st(out + off, ADD ? f4ld(out + off) + v : v);
}

// One query row of positive b: the dropped entity or relation row at triple column j, chunk (d, kp + d), and its masks
template <int HALVES>
struct DroppedRow {
    float4 re, im;
    Keep4 kr, ki;
    float scale;
    __device__ __forceinline__ DroppedRow(const OneVsAllSide &s, const SideDropout &dr, long long b, int j, int d)
    {
        const bool ent = j != 1;
        const uint32_t t = ent ? dr.t_ent : dr.t_rel;
        scale = ent ? dr.scale_ent : dr.scale_rel;
        const float *row = (ent ? s.ent : s.rel) + (size_t)s.triples[3 * b + j] * s.ld;
        const int tag = dropout_tag(s.side, 1 + j);
        kr = dropout_keep4(dr, b, d, tag, t);
        re = dropout_apply4(kr, f4ld(row + d), scale);
        if (HALVES == 2) {
            ki = dropout_keep4(dr, b, s.kp + d, tag, t);
            im = dropout_apply4(ki, f4ld(row + s.kp + d), scale);
        } else {
            ki = kr;
            im = f4zero();
        }
    }
};

// q[b] from the dropped query rows, one thread per (positive, float4 chunk of a half): side o Q1(s~, p~), side s
// Q0(p~, o~), side p Qp(s~, o~) = d f(s~, p, o~) / dp (scale excluded), with the training kernels' arithmetic
template <int HALVES>
__global__ void __launch_bounds__(256) kge_dropout_query_kernel(const OneVsAllSide s, const SideDropout dr, float *q)
{
    const int nq4 = s.kp / 4;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= s.B * nq4) return;
    const long long b = idx / nq4;
    const int d = (int)(idx - b * nq4) * 4;
    float *qb = q + (size_t)b * s.ld;
    const float4 z = f4zero();
    if (s.side == KGE_SIDE_O) {
        const DroppedRow<HALVES> sr(s, dr, b, 0, d), pr(s, dr, b, 1, d);
        f4st(qb + d, query_obj<HALVES, 0>(sr.re, sr.im, pr.re, pr.im));
        if (HALVES == 2) f4st(qb + s.kp + d, query_obj<HALVES, 1>(sr.re, sr.im, pr.re, pr.im));
    } else if (s.side == KGE_SIDE_S) {
        const DroppedRow<HALVES> pr(s, dr, b, 1, d), orr(s, dr, b, 2, d);
        f4st(qb + d, query_subj<HALVES, 0>(pr.re, pr.im, orr.re, orr.im));
        if (HALVES == 2) f4st(qb + s.kp + d, query_subj<HALVES, 1>(pr.re, pr.im, orr.re, orr.im));
    } else {
        const DroppedRow<HALVES> sr(s, dr, b, 0, d), orr(s, dr, b, 2, d);
        f4st(qb + d, trilinear_grad_p<HALVES, 0>(z, z, orr.re, orr.im, sr.re, sr.im, z, z));
        if (HALVES == 2) f4st(qb + s.kp + d, trilinear_grad_p<HALVES, 1>(z, z, orr.re, orr.im, sr.re, sr.im, z, z));
    }
}

// adds the raw gradient of one query row's chunk: (gr, gi) is the gradient of its dropped copy
template <int HALVES>
__device__ __forceinline__ void dropout_red(float *grad, const DroppedRow<HALVES> &r, int d, int kp, float4 gr, float4 gi)
{
    red_add_v4(grad + d, dropout_apply4(r.kr, gr, r.scale));
    if (HALVES == 2) red_add_v4(grad + kp + d, dropout_apply4(r.ki, gi, r.scale));
}

// The chain pass of kge_train_1vsall.cu (kge_ova_chain_kernel) on the dropped query rows: the same gradient rows of the
// query's two rows, formed from their dropped copies and masked before they are added
template <int HALVES>
__global__ void __launch_bounds__(256) kge_dropout_chain_kernel(const OneVsAllSide s, const SideDropout dr)
{
    const int nq4 = s.kp / 4;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= s.B * nq4) return;
    const long long b = idx / nq4;
    const int d = (int)(idx - b * nq4) * 4, di = HALVES == 2 ? s.kp + d : d;
    float4 Gr = f4zero(), Gi = f4zero();
    for (int k = 0; k < s.nsplit; ++k) {
        const float *g = s.pgq + ((size_t)k * s.B + b) * s.ld;
        Gr = Gr + f4ld(g + d);
        if (HALVES == 2) Gi = Gi + f4ld(g + di);
    }
    const int si = s.triples[3 * b], pi_ = s.triples[3 * b + 1], oi_ = s.triples[3 * b + 2];
    const float4 z = f4zero();
    float *gs_ = s.grad_ent + (size_t)si * s.ld, *go = s.grad_ent + (size_t)oi_ * s.ld;
    float *gp = s.grad_rel + (size_t)pi_ * s.ld;
    if (s.side == KGE_SIDE_P) {  // q = Qp(s, o): d/ds = Q0(Gq, o), d/do = Q1(s, Gq)
        const DroppedRow<HALVES> sr(s, dr, b, 0, d), orr(s, dr, b, 2, d);
        dropout_red<HALVES>(gs_, sr, d, s.kp, query_subj<HALVES, 0>(Gr, Gi, orr.re, orr.im),
                            HALVES == 2 ? query_subj<HALVES, 1>(Gr, Gi, orr.re, orr.im) : z);
        dropout_red<HALVES>(go, orr, d, s.kp, query_obj<HALVES, 0>(sr.re, sr.im, Gr, Gi),
                            HALVES == 2 ? query_obj<HALVES, 1>(sr.re, sr.im, Gr, Gi) : z);
        if (d == 0 && s.stamp_ent) {
            s.stamp_ent[si] = s.stamp;
            s.stamp_ent[oi_] = s.stamp;
        }
        return;
    }
    if (s.side == KGE_SIDE_O) {  // q = Q1(s, p): d/ds = Q0(p, Gq), d/dp of f(s, p, Gq)
        const DroppedRow<HALVES> sr(s, dr, b, 0, d), pr(s, dr, b, 1, d);
        dropout_red<HALVES>(gs_, sr, d, s.kp, query_subj<HALVES, 0>(pr.re, pr.im, Gr, Gi),
                            HALVES == 2 ? query_subj<HALVES, 1>(pr.re, pr.im, Gr, Gi) : z);
        dropout_red<HALVES>(gp, pr, d, s.kp, trilinear_grad_p<HALVES, 0>(sr.re, sr.im, z, z, z, z, Gr, Gi),
                            HALVES == 2 ? trilinear_grad_p<HALVES, 1>(sr.re, sr.im, z, z, z, z, Gr, Gi) : z);
    } else {  // q = Q0(p, o): d/do = Q1(Gq, p), d/dp of f(Gq, p, o)
        const DroppedRow<HALVES> pr(s, dr, b, 1, d), orr(s, dr, b, 2, d);
        dropout_red<HALVES>(go, orr, d, s.kp, query_obj<HALVES, 0>(Gr, Gi, pr.re, pr.im),
                            HALVES == 2 ? query_obj<HALVES, 1>(Gr, Gi, pr.re, pr.im) : z);
        dropout_red<HALVES>(gp, pr, d, s.kp, trilinear_grad_p<HALVES, 0>(z, z, orr.re, orr.im, Gr, Gi, z, z),
                            HALVES == 2 ? trilinear_grad_p<HALVES, 1>(z, z, orr.re, orr.im, Gr, Gi, z, z) : z);
    }
    if (d == 0 && s.stamp_rel) s.stamp_rel[pi_] = s.stamp;
}

static unsigned grid_of(long long n) { return (unsigned)((n + 255) / 256); }

cudaError_t launch_dropout_prepare(OneVsAllSide &s, const SideDropout &d, float *q, int halves, cudaStream_t st)
{
    const bool rel = s.side == KGE_SIDE_P;
    const int tag = dropout_tag(s.side, 0);
    kge_dropout_rows_kernel<false><<<grid_of(s.n_cand * (s.ld / 4)), 256, 0, st>>>(
        s.cand, d.cand, s.n_cand, s.ld, d, tag, rel ? d.t_rel : d.t_ent, rel ? d.scale_rel : d.scale_ent);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(d.grad_cand, 0, (size_t)s.n_cand * s.ld * sizeof(float), st)) != cudaSuccess) return e;
    const unsigned grid = grid_of(s.B * (s.kp / 4));
    if (halves == 2) kge_dropout_query_kernel<2><<<grid, 256, 0, st>>>(s, d, q);
    else kge_dropout_query_kernel<1><<<grid, 256, 0, st>>>(s, d, q);
    s.cand = d.cand;
    s.grad_cand = d.grad_cand;
    s.q = q;
    return cudaGetLastError();
}

cudaError_t launch_dropout_finish(const OneVsAllSide &s, const SideDropout &d, int halves, cudaStream_t st)
{
    const bool rel = s.side == KGE_SIDE_P;
    kge_dropout_rows_kernel<true><<<grid_of(s.n_cand * (s.ld / 4)), 256, 0, st>>>(
        d.grad_cand, rel ? s.grad_rel : s.grad_ent, s.n_cand, s.ld, d, dropout_tag(s.side, 0), rel ? d.t_rel : d.t_ent,
        rel ? d.scale_rel : d.scale_ent);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    const unsigned grid = grid_of(s.B * (s.kp / 4));
    if (halves == 2) kge_dropout_chain_kernel<2><<<grid, 256, 0, st>>>(s, d);
    else kge_dropout_chain_kernel<1><<<grid, 256, 0, st>>>(s, d);
    return cudaGetLastError();
}

}  // namespace kge
