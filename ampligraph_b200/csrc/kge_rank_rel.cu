// kge_rank_rel.cu -- relation prediction (s, ?, o): score every test triple's (s, o) pair against every candidate
// relation and count ranks (sm_90a).
//
// The candidates of this side are relation rows, so every (query, candidate) pair has its own query vector: the
// per-query qvec staging of kge_rank.cu does not apply.  The score of (s, r, o) is the canonical triple score of
// oracle/kge_oracle.c: kgeo_score_triple, the value kge_rank quantises as a positive's score (launch_rank_prepare):
//   TransE / DistMult / RotatE: the object-side chain with candidate o, its query vector built from (s, r) with the
//     operations of kge_rank_qvec_kernel (s + p, s * p, the rotated subject);
//   ComplEx / HolE: the subject-side chain with candidate s, its query vector built from (r, o).
// Each step below builds one column of that vector and feeds it to rank_step / rank_step_rot of kge_rank_common.cuh,
// so the count kernel and the filter kernel run the same operations in the same order as the positive.
#include "kge_rank_common.cuh"

namespace kge {

// The chain of the relation side: M is the model, HolE runs as KGE_COMPLEX (its scale is applied by rank_finish)
template <int M>
__host__ __device__ constexpr int rel_op() { return M == KGE_TRANSE ? OP_L1_SUB : M == KGE_ROTATE ? OP_ROT_O : OP_DOT; }

// one column of a single-half row (TransE: q = s + p, acc + |q - o|; DistMult: q = s * p, fma(o, q, acc))
template <int M>
__device__ __forceinline__ float rel_step(float acc, float s, float p, float o)
{
    if (M == KGE_TRANSE) return rank_step<OP_L1_SUB>(acc, o, __fadd_rn(s, p));
    return rank_step<OP_DOT>(acc, o, __fmul_rn(s, p));
}
// one column d of the real (IM = false) or imaginary (IM = true) half of ComplEx / HolE: q = (r, o)'s subject-side
// query vector (ComplEx.py:95-106), fma(s, q, acc)
template <bool IM>
__device__ __forceinline__ float rel_step_cplx(float acc, float s_h, float pr, float pi, float o_re, float o_im)
{
    const float q = IM ? __fmaf_rn(-pi, o_re, __fmul_rn(pr, o_im)) : __fmaf_rn(pi, o_im, __fmul_rn(pr, o_re));
    return rank_step<OP_DOT>(acc, s_h, q);
}
// one column d of RotatE: (c, sn) = the relation's rotation, q = the rotated subject (RotatE.py:208-211), |q - o|
__device__ __forceinline__ float rel_step_rot(float acc, float s_re, float s_im, float c, float sn, float o_re, float o_im)
{
    const float qa = __fmaf_rn(-s_im, sn, __fmul_rn(s_re, c)), qb = __fmaf_rn(s_im, c, __fmul_rn(s_re, sn));
    return rank_step_rot<OP_ROT_O>(acc, o_re, o_im, qa, qb, 0.f, 0.f);
}

// The whole chain of one pair from its three rows (kp floats per half, ld per row)
template <int M>
__device__ __forceinline__ float rel_score(const float *s, const float *p, const float *o, int kp, int ld, float scale)
{
    float acc = 0.f;
    if (M == KGE_TRANSE || M == KGE_DISTMULT) {
#pragma unroll 8
        for (int d = 0; d < ld; ++d) acc = rel_step<M>(acc, s[d], p[d], o[d]);
    } else if (M == KGE_ROTATE) {
#pragma unroll 4
        for (int d = 0; d < kp; ++d) acc = rel_step_rot(acc, s[d], s[kp + d], p[d], p[kp + d], o[d], o[kp + d]);
    } else {
#pragma unroll 4
        for (int d = 0; d < kp; ++d) acc = rel_step_cplx<false>(acc, s[d], p[d], p[kp + d], o[d], o[kp + d]);
#pragma unroll 4
        for (int d = 0; d < kp; ++d) acc = rel_step_cplx<true>(acc, s[kp + d], p[d], p[kp + d], o[d], o[kp + d]);
    }
    return rank_finish<rel_op<M>()>(acc, scale);
}

// --------------------------------------------------------------------------
// count kernel: CTA = 32 queries x 64 candidate relations, 8 warps; lane = query, warp w = relations 8w .. 8w + 7, one
// chain per accumulator register.  Per column chunk the CTA stages the s and o rows of its queries and the rows of its
// relations with cp.async (16 B, zero-fill past the row end or the last query / candidate), double buffered; a chunk is
// 32 columns of a single-half row, or 16 columns of each half (re | im) of a two-half row.  ComplEx / HolE walk the
// chunks twice: the canonical chain adds every real column before the first imaginary one.  Rows are padded to 36 floats:
// the lanes' 128-bit reads of their own query rows are bank-conflict free, the relation reads are broadcasts.
// --------------------------------------------------------------------------
constexpr int RL_TQ = 32, RL_TR = 64, RL_RPW = 8, RL_DK = 32, RL_LDS = RL_DK + 4, RL_THREADS = 256;
constexpr int RL_Q_FLOATS = RL_TQ * RL_LDS, RL_R_FLOATS = RL_TR * RL_LDS;
constexpr int RL_STAGE_FLOATS = 2 * RL_Q_FLOATS + RL_R_FLOATS;

template <int M>
__global__ void __launch_bounds__(RL_THREADS, 2) kge_rank_rel_kernel(const RankParams p, const float *__restrict__ rel,
                                                                     const int32_t *__restrict__ triples, int32_t *__restrict__ cnt)
{
    constexpr bool HALVES = M != KGE_TRANSE && M != KGE_DISTMULT;
    extern __shared__ __align__(128) float smem[];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const long long q0 = (long long)blockIdx.y * RL_TQ, c0 = (long long)blockIdx.x * RL_TR;
    const int ld = p.L.ld, kp = p.L.kp;
    const int n_chunks = HALVES ? (kp + 15) / 16 : (ld + RL_DK - 1) / RL_DK;
    const int n_iter = M == KGE_COMPLEX ? 2 * n_chunks : n_chunks;

    // staging: thread t copies column quad t%8 of query row t/8 (its s and o rows) and of relation rows t/8, t/8 + 32
    const int lrow = t >> 3, c4 = t & 7;
    const long long q = q0 + lrow;
    const bool qvalid = q < p.b;
    const float *srow = p.ent + (size_t)(qvalid ? triples[3 * q] : 0) * ld;
    const float *orow = p.ent + (size_t)(qvalid ? triples[3 * q + 2] : 0) * ld;
    const float *rrow[2];
    bool rvalid[2];
#pragma unroll
    for (int n = 0; n < 2; ++n) {
        const long long c = c0 + lrow + 32 * n;
        rvalid[n] = c < p.n_cand;
        const long long id = rvalid[n] ? (p.cand_ids ? (long long)p.cand_ids[c] : p.cand_begin + c) : 0;
        rrow[n] = rel + (size_t)id * ld;
    }

    auto stage_load = [&](int it, int buf) {
        float *Ss = smem + buf * RL_STAGE_FLOATS, *Os = Ss + RL_Q_FLOATS, *Rs = Os + RL_Q_FLOATS;
        const int chunk = it % n_chunks;
        const int d = HALVES ? chunk * 16 + 4 * (c4 & 3) : chunk * RL_DK + 4 * c4;
        const bool cvalid = d < (HALVES ? kp : ld);
        const int col = cvalid ? (HALVES && c4 >= 4 ? kp : 0) + d : 0;
        const int so = lrow * RL_LDS + 4 * c4;
        cp_async16(Ss + so, srow + col, cvalid && qvalid);
        cp_async16(Os + so, orow + col, cvalid && qvalid);
#pragma unroll
        for (int n = 0; n < 2; ++n) cp_async16(Rs + so + 32 * n * RL_LDS, rrow[n] + col, cvalid && rvalid[n]);
        cp_async_commit();
    };

    float acc[RL_RPW];
#pragma unroll
    for (int m = 0; m < RL_RPW; ++m) acc[m] = 0.f;

    stage_load(0, 0);
    for (int it = 0; it < n_iter; ++it) {
        const int buf = it & 1;
        if (it + 1 < n_iter) {
            stage_load(it + 1, buf ^ 1);
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        const float *Ss = smem + buf * RL_STAGE_FLOATS + lane * RL_LDS, *Os = Ss + RL_Q_FLOATS;
        const float *Rs = smem + buf * RL_STAGE_FLOATS + 2 * RL_Q_FLOATS + warp * RL_RPW * RL_LDS;
        if constexpr (!HALVES) {
#pragma unroll
            for (int d4 = 0; d4 < RL_DK / 4; ++d4) {
                const float4 s = *reinterpret_cast<const float4 *>(Ss + 4 * d4), o = *reinterpret_cast<const float4 *>(Os + 4 * d4);
#pragma unroll
                for (int m = 0; m < RL_RPW; ++m) {
                    const float4 r = *reinterpret_cast<const float4 *>(Rs + m * RL_LDS + 4 * d4);
                    float a = acc[m];
                    a = rel_step<M>(a, s.x, r.x, o.x);
                    a = rel_step<M>(a, s.y, r.y, o.y);
                    a = rel_step<M>(a, s.z, r.z, o.z);
                    a = rel_step<M>(a, s.w, r.w, o.w);
                    acc[m] = a;
                }
            }
        } else {
            const bool im = M == KGE_COMPLEX && it >= n_chunks;  // ComplEx / HolE: second walk, the imaginary half
#pragma unroll
            for (int d4 = 0; d4 < 4; ++d4) {
                const float4 sr = *reinterpret_cast<const float4 *>(Ss + 4 * d4), si = *reinterpret_cast<const float4 *>(Ss + 16 + 4 * d4);
                const float4 orr = *reinterpret_cast<const float4 *>(Os + 4 * d4), oi = *reinterpret_cast<const float4 *>(Os + 16 + 4 * d4);
#pragma unroll
                for (int m = 0; m < RL_RPW; ++m) {
                    const float4 pr = *reinterpret_cast<const float4 *>(Rs + m * RL_LDS + 4 * d4);
                    const float4 pi = *reinterpret_cast<const float4 *>(Rs + m * RL_LDS + 16 + 4 * d4);
                    float a = acc[m];
                    if (M == KGE_ROTATE) {
                        a = rel_step_rot(a, sr.x, si.x, pr.x, pi.x, orr.x, oi.x);
                        a = rel_step_rot(a, sr.y, si.y, pr.y, pi.y, orr.y, oi.y);
                        a = rel_step_rot(a, sr.z, si.z, pr.z, pi.z, orr.z, oi.z);
                        a = rel_step_rot(a, sr.w, si.w, pr.w, pi.w, orr.w, oi.w);
                    } else if (im) {
                        a = rel_step_cplx<true>(a, si.x, pr.x, pi.x, orr.x, oi.x);
                        a = rel_step_cplx<true>(a, si.y, pr.y, pi.y, orr.y, oi.y);
                        a = rel_step_cplx<true>(a, si.z, pr.z, pi.z, orr.z, oi.z);
                        a = rel_step_cplx<true>(a, si.w, pr.w, pi.w, orr.w, oi.w);
                    } else {
                        a = rel_step_cplx<false>(a, sr.x, pr.x, pi.x, orr.x, oi.x);
                        a = rel_step_cplx<false>(a, sr.y, pr.y, pi.y, orr.y, oi.y);
                        a = rel_step_cplx<false>(a, sr.z, pr.z, pi.z, orr.z, oi.z);
                        a = rel_step_cplx<false>(a, sr.w, pr.w, pi.w, orr.w, oi.w);
                    }
                    acc[m] = a;
                }
            }
        }
        __syncthreads();
    }

    // count epilogue (kge_rank.cu: count_tile, with the query on the lane): quantise, compare with the positive, count
    // the greater and the equal candidates; with p.scores set, store every score as well
    const long long qi = q0 + lane;
    const bool qok = qi < p.b;
    const int qp = qok ? p.qpos[qi] : 0;
    int gt = 0, eq = 0;
#pragma unroll
    for (int m = 0; m < RL_RPW; ++m) {
        const long long c = c0 + warp * RL_RPW + m;
        const bool cok = c < p.n_cand;
        const float sc = rank_finish<rel_op<M>()>(acc[m], p.scale);
        if (p.scores && qok && cok) p.scores[(size_t)qi * p.n_cand + c] = sc;
        const int qc = quantise(sc);
        gt += (cok && qp < qc) ? 1 : 0;
        eq += (cok && qp == qc) ? 1 : 0;
    }
    if (qok) {
        if (gt) atomicAdd(&cnt[3 * qi + 0], gt);
        if (eq) atomicAdd(&cnt[3 * qi + 1], eq);
    }
}

// --------------------------------------------------------------------------
// filter kernel: the filter walk on the relation side, each (query, known-true relation) pair scored by rel_score from
// its staged s, relation and o rows
// --------------------------------------------------------------------------
template <int M>
__global__ void kge_rank_rel_filter_kernel(const RankParams p, const float *__restrict__ rel, const int32_t *__restrict__ triples,
                                           const long long *__restrict__ off, const int32_t *__restrict__ idx,
                                           int32_t *__restrict__ cnt)
{
    extern __shared__ __align__(16) float pair_sm[];
    const int lane = threadIdx.x & 31, ld = p.L.ld;
    float *sm = pair_sm + (size_t)(threadIdx.x >> 5) * 3 * ld;
    filter_walk(p, off, idx, cnt, [&](long long i, long long id) {
        return warp_chain<3>(p.ent + (size_t)triples[3 * i] * ld, rel + (size_t)id * ld, p.ent + (size_t)triples[3 * i + 2] * ld, ld,
                             sm, lane, [&](const float *s, const float *r, const float *o) {
                                 return rel_score<M>(s, r, o, p.L.kp, ld, p.scale);
                             });
    });
}

// Host side: launch(std::integral_constant<int, M>) for the model's relation-side kernel instance; HolE runs ComplEx's
template <class Launch>
static cudaError_t dispatch_rel_model(int model, Launch &&launch)
{
    return dispatch_value<KGE_TRANSE, KGE_DISTMULT, KGE_COMPLEX, KGE_ROTATE>(model == KGE_HOLE ? KGE_COMPLEX : model, launch);
}

cudaError_t launch_rank_rel_count(const RankParams &p, const float *rel, const int32_t *triples, int32_t *cnt, cudaStream_t st)
{
    if (p.b == 0 || p.n_cand == 0) return cudaSuccess;
    const dim3 grid((unsigned)((p.n_cand + RL_TR - 1) / RL_TR), (unsigned)((p.b + RL_TQ - 1) / RL_TQ));
    return dispatch_rel_model(p.L.model, [&](auto m) {
        return launch_with_smem(kge_rank_rel_kernel<decltype(m)::value>, grid, RL_THREADS, 2 * RL_STAGE_FLOATS * sizeof(float),
                                st, p, rel, triples, cnt);
    });
}

cudaError_t launch_rank_rel_filter(const RankParams &p, const float *rel, const int32_t *triples, const long long *filt_off,
                                   const int32_t *filt_idx, long long n_pairs, int32_t *cnt, int sm_count, cudaStream_t st)
{
    if (n_pairs == 0 || p.b == 0) return cudaSuccess;
    const PairLaunch pl = pair_launch(p.L.ld, 3);
    const long long want = (n_pairs + pl.warps - 1) / pl.warps;
    const unsigned grid = (unsigned)(want < (long long)sm_count * 8 ? want : (long long)sm_count * 8);
    return dispatch_rel_model(p.L.model, [&](auto m) {
        return launch_with_smem(kge_rank_rel_filter_kernel<decltype(m)::value>, grid, pl.warps * 32, pl.smem, st, p, rel, triples,
                                filt_off, filt_idx, cnt);
    });
}

}  // namespace kge
