// kge_train_shared.cu -- sampled training with shared negatives (kge_shared_negatives_step, DESIGN.md 3.21; sm_90a).
//
// A step's B positives are cut into chunks of C consecutive positives; every positive of chunk k is corrupted with the
// same eta candidate entities c_{k,j} = draw_corruption's replacement for r = j*B + k*C, so a candidate row is read
// once per chunk slice instead of once per positive.  The side of corruption (i, j) is the per-positive sampler's side
// for r = j*B + i (fair coin, or the Bernoulli threshold of the positive's relation).
//
// Three passes over a caller-owned workspace ([B, eta] scores, [B, eta] side bytes, [B] positive scores):
//   score     one CTA per (chunk, tile of 32 candidates, slice of 16 positives).  The tile's candidate rows are
//             staged in shared memory with cp.async, one column window of 128 floats per half at a time (so rows of
//             any width fit); each warp scores its positives against the 32 staged rows, lane t keeping candidate t's
//             running score across the windows.  The tile-0 CTAs also score the positives.
//   loss      one warp per positive: loss_and_dscores in place on its row of scores (the fused step's loss code).
//   gradient  the score pass's grid again.  Each warp forms g * d score / d candidate for its positives and adds it to
//             the tile's gradient rows in shared memory; after every window the CTA adds each candidate row to
//             grad_ent once (one red.global.add.v4 per float4).  The kept rows' terms go straight to grad_ent /
//             grad_rel as in the general kernel's finish, with the positive's own dL/dscore added by the tile-0 CTA.
// The per-pair arithmetic is kge_train_common.cuh's (query_subj / query_obj / trilinear_grad_p, rot_*) and the
// general kernel's TransE distance and sign arithmetic, one float4 chunk per lane and half.
#include "kge_train_common.cuh"

namespace kge {

namespace {

constexpr int SN_TJ = 32;        // candidates per tile (lane t holds candidate t's score)
constexpr int SN_WK = 128;       // floats per half of a column window: one float4 per lane
constexpr int SN_WARPS = 8;      // warps per CTA of the score and gradient passes
constexpr int SN_PPW = 2;        // positives per warp of one CTA
constexpr int SN_PS = SN_WARPS * SN_PPW;  // positives per CTA (chunk slice)

struct Tile {
    long long i_begin, i_end;  // the CTA's positives
    int j0, nt;                // its candidates [j0, j0 + nt)
    bool first;                // the tile of candidates 0..31: adds the positives' own terms
};

__device__ __forceinline__ Tile tile_of(const SharedNegParams &q)
{
    const long long bid = blockIdx.x;
    const int jt = (int)(bid % q.n_jt);
    const long long rest = bid / q.n_jt;
    const long long ps = rest % q.n_ps, k = rest / q.n_ps;
    const long long c0 = k * q.chunk, c1 = min(c0 + q.chunk, q.t.B);
    Tile t;
    t.i_begin = c0 + ps * SN_PS;
    t.i_end = min(t.i_begin + SN_PS, c1);
    t.j0 = jt * SN_TJ;
    t.nt = min(SN_TJ, q.t.eta - t.j0);
    t.first = jt == 0;
    return t;
}

// the chunk's candidates of the tile (entity ids) into cid[0, nt)
__device__ __forceinline__ void tile_candidates(const SharedNegParams &q, const Tile &t, int *cid, bool stamp)
{
    const long long k = t.i_begin / q.chunk;
    if ((int)threadIdx.x < t.nt) {
        int keep, repl;
        const unsigned long long r = (unsigned long long)(t.j0 + threadIdx.x) * (unsigned long long)q.t.B +
                                     (unsigned long long)(k * q.chunk);
        draw_corruption(q.t.seed, q.t.step, r, q.t.n_ent, &keep, &repl);
        cid[threadIdx.x] = repl;
        if (stamp && q.t.stamp_ent) q.t.stamp_ent[repl] = q.t.stamp;
    }
}

// side of corruption (i, j): 1 = subject kept, object replaced (the sampler's keep_subj for r = j*B + i)
__device__ __forceinline__ int pair_side(const SharedNegParams &q, long long i, int j, int rel)
{
    const unsigned long long r = (unsigned long long)j * (unsigned long long)q.t.B + (unsigned long long)i;
    const u32x4 v = philox4x32_10((uint32_t)r, (uint32_t)(r >> 32), (uint32_t)q.t.step, (uint32_t)(q.t.step >> 32),
                                  (uint32_t)q.t.seed, (uint32_t)(q.t.seed >> 32));
    return q.thr ? (v.x >= q.thr[rel] ? 1 : 0) : (int)(v.x & 1u);
}

// window cb of the tile's candidate rows into cand[t][h * SN_WK + c] (zero past the half's end)
template <int HALVES>
__device__ __forceinline__ void stage_window(const SharedNegParams &q, const int *cid, int nt, int cb, float *cand)
{
    const int nch = q.t.kp / 4;
    for (int x = threadIdx.x; x < nt * HALVES * 32; x += blockDim.x) {
        const int c = x & 31, h = (x >> 5) % HALVES, t = (x >> 5) / HALVES;
        const int col = cb * 32 + c;
        const bool valid = col < nch;
        const float *src = q.t.ent + (size_t)cid[t] * q.t.ld + h * q.t.kp + (valid ? 4 * col : 0);
        cp_async16(cand + (t * HALVES + h) * SN_WK + 4 * c, src, valid);
    }
    cp_async_commit();
    cp_async_wait<0>();
}

// ---- per-model pair arithmetic on one float4 chunk per half (x[0]: re / only half, x[1]: im) ----
template <int MODEL>
struct PairOps;

// DistMult / ComplEx / HolE (HALVES 1 / 2): the score of a corruption is <row, Q>
template <int HALVES>
struct TrilinearOps {
    float4 s[2], p[2], o[2], A[2], Cq[2], Ws[2], Wo[2];
    __device__ __forceinline__ void load(const float *sr, const float *pr, const float *orow, int off, int kp, bool live)
    {
#pragma unroll
        for (int h = 0; h < HALVES; ++h) {
            s[h] = live ? f4ld(sr + h * kp + off) : f4zero();
            p[h] = live ? f4ld(pr + h * kp + off) : f4zero();
            o[h] = live ? f4ld(orow + h * kp + off) : f4zero();
            Ws[h] = Wo[h] = f4zero();
        }
        if constexpr (HALVES == 1) {
            A[0] = query_subj<1, 0>(p[0], p[0], o[0], o[0]);
            Cq[0] = query_obj<1, 0>(s[0], s[0], p[0], p[0]);
        } else {
            query_subj<2>(p[0], p[1], o[0], o[1], A[0], A[1]);
            query_obj<2>(s[0], s[1], p[0], p[1], Cq[0], Cq[1]);
        }
    }
    __device__ __forceinline__ float dot(const float4 *q, const float4 *r) const
    {
        float4 a = f4fma(r[0], q[0], f4zero());
        if constexpr (HALVES == 2) a = f4fma(r[1], q[1], a);
        return f4hsum(a);
    }
    __device__ __forceinline__ float positive() const { return dot(A, s); }
    template <int SIDE>
    __device__ __forceinline__ float partial(const float4 *r) const { return dot(SIDE ? Cq : A, r); }
    template <int SIDE>
    __device__ __forceinline__ void grad(const float4 *r, float g, float4 *out)
    {
#pragma unroll
        for (int h = 0; h < HALVES; ++h) {
            float4 &W = SIDE ? Wo[h] : Ws[h];
            W = f4fma(g, r[h], W);
            out[h] = g * (SIDE ? Cq[h] : A[h]);
        }
    }
    // gradient chunks of the kept rows (the general kernel's finish): gs, gp, go per half
    __device__ __forceinline__ void finish(float gP, float, float4 *gs, float4 *gp, float4 *go) const
    {
        if constexpr (HALVES == 1) {
            const float4 U = f4fma(gP, s[0], Ws[0]), X = f4fma(gP, o[0], Wo[0]);
            gs[0] = query_subj<1, 0>(p[0], p[0], X, X);
            go[0] = query_obj<1, 0>(U, U, p[0], p[0]);
            gp[0] = trilinear_grad_p<1, 0>(s[0], s[0], o[0], o[0], U, U, Wo[0], Wo[0]);
        } else {
            const float4 Ur = f4fma(gP, s[0], Ws[0]), Ui = f4fma(gP, s[1], Ws[1]);
            const float4 Xr = f4fma(gP, o[0], Wo[0]), Xi = f4fma(gP, o[1], Wo[1]);
            gs[0] = query_subj<2, 0>(p[0], p[1], Xr, Xi);
            gs[1] = query_subj<2, 1>(p[0], p[1], Xr, Xi);
            go[0] = query_obj<2, 0>(Ur, Ui, p[0], p[1]);
            go[1] = query_obj<2, 1>(Ur, Ui, p[0], p[1]);
            gp[0] = trilinear_grad_p<2, 0>(s[0], s[1], o[0], o[1], Ur, Ui, Wo[0], Wo[1]);
            gp[1] = trilinear_grad_p<2, 1>(s[0], s[1], o[0], o[1], Ur, Ui, Wo[0], Wo[1]);
        }
    }
};
template <> struct PairOps<KGE_DISTMULT> : TrilinearOps<1> {};
template <> struct PairOps<KGE_COMPLEX> : TrilinearOps<2> {};
template <> struct PairOps<KGE_HOLE> : TrilinearOps<2> {};

// TransE: f = -sum |s + p - o|
template <>
struct PairOps<KGE_TRANSE> {
    float4 o, Qs, Qo, Vs, Vo;  // p - o, s + p, sum g * sign per side
    __device__ __forceinline__ void load(const float *sr, const float *pr, const float *orow, int off, int, bool live)
    {
        const float4 vs = live ? f4ld(sr + off) : f4zero(), vp = live ? f4ld(pr + off) : f4zero();
        o = live ? f4ld(orow + off) : f4zero();
        Qs = vp - o;
        Qo = vs + vp;
        Vs = Vo = f4zero();
    }
    __device__ __forceinline__ float positive() const { return -f4abssum(Qo - o); }
    template <int SIDE>
    __device__ __forceinline__ float partial(const float4 *r) const { return -f4abssum(SIDE ? (Qo - r[0]) : (r[0] + Qs)); }
    template <int SIDE>
    __device__ __forceinline__ void grad(const float4 *r, float g, float4 *out)
    {
        // SIDE 1: t = (s+p) - r, df/dr = +sign(t);  SIDE 0: t = r + (p-o), df/dr = -sign(t)
        const float4 sa = g * f4sgn(SIDE ? (Qo - r[0]) : (r[0] + Qs));
        float4 &V = SIDE ? Vo : Vs;
        V = V + sa;
        out[0] = SIDE ? sa : f4neg(sa);
    }
    __device__ __forceinline__ void finish(float gP, float, float4 *gs, float4 *gp, float4 *go) const
    {
        const float4 Vp = gP * f4sgn(Qo - o);
        gs[0] = f4neg(Vp + Vo);
        gp[0] = f4neg(Vp + Vs + Vo);
        go[0] = Vp + Vs;
    }
};

// RotatE: the relation row is the rotation table row [cos(phi) | sin(phi)]
template <>
struct PairOps<KGE_ROTATE> {
    float4 C, Sn, Or, Oi, Yr, Yi, Zor, Zoi, Zsr, Zsi, Aphi;
    __device__ __forceinline__ void load(const float *sr, const float *pr, const float *orow, int off, int kp, bool live)
    {
        const float4 s0 = live ? f4ld(sr + off) : f4zero(), s1 = live ? f4ld(sr + kp + off) : f4zero();
        C = live ? f4ld(pr + off) : f4zero();
        Sn = live ? f4ld(pr + kp + off) : f4zero();
        Or = live ? f4ld(orow + off) : f4zero();
        Oi = live ? f4ld(orow + kp + off) : f4zero();
        Yr = rot_rotate<0>(s0, s1, C, Sn);
        Yi = rot_rotate<1>(s0, s1, C, Sn);
        Zor = Zoi = Zsr = Zsi = Aphi = f4zero();
    }
    __device__ __forceinline__ float positive() const { return -rot_modsum(Yr - Or, Yi - Oi); }
    template <int SIDE>
    __device__ __forceinline__ float partial(const float4 *r) const
    {
        if (SIDE) return -rot_modsum(Yr - r[0], Yi - r[1]);
        return -rot_modsum(rot_residual_subj<0>(r[0], r[1], C, Sn, Or, Oi), rot_residual_subj<1>(r[0], r[1], C, Sn, Or, Oi));
    }
    template <int SIDE>
    __device__ __forceinline__ void grad(const float4 *r, float g, float4 *out)
    {
        float4 a, b;
        if (SIDE) {  // residual = y(s) - r ; df/dr = +(a,b)
            rot_unit(Yr - r[0], Yi - r[1], g, a, b);
            Zor = Zor + a; Zoi = Zoi + b;
            out[0] = a; out[1] = b;
        } else {  // residual = R(phi) r - o ; df/dr = -R(-phi)(a,b)
            const float4 yr = rot_rotate<0>(r[0], r[1], C, Sn), yi = rot_rotate<1>(r[0], r[1], C, Sn);
            rot_unit(yr - Or, yi - Oi, g, a, b);
            Zsr = Zsr + a; Zsi = Zsi + b;
            Aphi = rot_dphi(a, b, yr, yi, Aphi);
            out[0] = rot_back<0>(a, b, C, Sn);
            out[1] = rot_back<1>(a, b, C, Sn);
        }
    }
    // the relation row receives d/dtheta = (1/div) d/dphi in its first half only (gp[1] is not added)
    __device__ __forceinline__ void finish(float gP, float inv_div, float4 *gs, float4 *gp, float4 *go) const
    {
        float4 a, b;
        rot_unit(Yr - Or, Yi - Oi, gP, a, b);
        const float4 Zr = a + Zor, Zi = b + Zoi;
        gs[0] = rot_back<0>(Zr, Zi, C, Sn);
        gs[1] = rot_back<1>(Zr, Zi, C, Sn);
        go[0] = a + Zsr;
        go[1] = b + Zsi;
        gp[0] = inv_div * rot_dphi(Zr, Zi, Yr, Yi, Aphi);
        gp[1] = f4zero();
    }
};

template <int MODEL>
__device__ __forceinline__ void read_row(const float *cand, int t, float4 *r)
{
    constexpr int HALVES = (MODEL == KGE_TRANSE || MODEL == KGE_DISTMULT) ? 1 : 2;
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int h = 0; h < HALVES; ++h) r[h] = f4ld(cand + (t * HALVES + h) * SN_WK + 4 * lane);
}

// ---- pass 1: scores -> sc[i * eta + j], the positive's score -> pos[i], sides -> keep[i * eta + j] ----
template <int MODEL>
__global__ void __launch_bounds__(SN_WARPS * 32) kge_shared_scores_kernel(const SharedNegParams q)
{
    constexpr int HALVES = (MODEL == KGE_TRANSE || MODEL == KGE_DISTMULT) ? 1 : 2;
    __shared__ __align__(16) float cand[SN_TJ * HALVES * SN_WK];
    __shared__ int cid[SN_TJ];
    const Tile t = tile_of(q);
    if (t.i_begin >= t.i_end) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int eta = q.t.eta, kp = q.t.kp, ld = q.t.ld, nch = kp / 4, n_cb = (kp + SN_WK - 1) / SN_WK;
    const bool stamps = q.t.stamp_ent != nullptr;
    tile_candidates(q, t, cid, stamps && t.i_begin % q.chunk == 0);

    float acc[SN_PPW], pacc[SN_PPW];
    unsigned side1[SN_PPW];
#pragma unroll
    for (int u = 0; u < SN_PPW; ++u) {
        acc[u] = pacc[u] = 0.f;
        side1[u] = 0u;
        const long long i = t.i_begin + warp + SN_WARPS * u;
        if (i < t.i_end) {
            const int rel = q.t.triples[3 * i + 1];
            const int keep = lane < t.nt ? pair_side(q, i, t.j0 + lane, rel) : 0;
            if (lane < t.nt) q.keep[i * eta + t.j0 + lane] = (uint8_t)keep;
            side1[u] = __ballot_sync(0xffffffffu, keep != 0);
            if (t.first && stamps) {
                if (lane == 0) q.t.stamp_ent[q.t.triples[3 * i]] = q.t.stamp;
                if (lane == 1) q.t.stamp_ent[q.t.triples[3 * i + 2]] = q.t.stamp;
                if (lane == 2 && q.t.stamp_rel) q.t.stamp_rel[rel] = q.t.stamp;
            }
        }
    }
    __syncthreads();
    for (int cb = 0; cb < n_cb; ++cb) {
        stage_window<HALVES>(q, cid, t.nt, cb, cand);
        __syncthreads();
        const int col = cb * 32 + lane;
        const bool live = col < nch;
#pragma unroll
        for (int u = 0; u < SN_PPW; ++u) {
            const long long i = t.i_begin + warp + SN_WARPS * u;
            if (i >= t.i_end) continue;
            const int s_id = q.t.triples[3 * i], p_id = q.t.triples[3 * i + 1], o_id = q.t.triples[3 * i + 2];
            PairOps<MODEL> S;
            S.load(q.t.ent + (size_t)s_id * ld, q.t.rel + (size_t)p_id * ld, q.t.ent + (size_t)o_id * ld, 4 * col, kp, live);
            if (t.first) pacc[u] += warp_sum(S.positive());
            for (int c = 0; c < t.nt; ++c) {
                float4 r[2];
                read_row<MODEL>(cand, c, r);
                const float v = warp_sum(((side1[u] >> c) & 1u) ? S.template partial<1>(r) : S.template partial<0>(r));
                if (lane == c) acc[u] += v;
            }
        }
        __syncthreads();
    }
#pragma unroll
    for (int u = 0; u < SN_PPW; ++u) {
        const long long i = t.i_begin + warp + SN_WARPS * u;
        if (i >= t.i_end) continue;
        if (lane < t.nt) q.sc[i * eta + t.j0 + lane] = acc[u];
        if (t.first && lane == 0) q.pos[i] = pacc[u];
    }
}

// ---- pass 2: loss and dL/dscore in place: sc[i, :] -> dL/dN (unscaled), pos[i] -> dL/dP ----
__global__ void __launch_bounds__(256) kge_shared_loss_kernel(const SharedNegParams q)
{
    const int lane = threadIdx.x & 31;
    const long long n_warps = (long long)gridDim.x * (blockDim.x >> 5);
    const float scale = q.t.score_scale;
    double loss_acc = 0.0;
    for (long long i = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); i < q.t.B; i += n_warps) {
        float *sc = q.sc + i * q.t.eta;
        if (scale != 1.f)
            for (int j = lane; j < q.t.eta; j += 32) sc[j] *= scale;
        __syncwarp();
        float dP;
        const float li = loss_and_dscores(q.t, scale * q.pos[i], sc, lane, &dP);
        if (lane == 0) { loss_acc += (double)li; q.pos[i] = dP; }
        __syncwarp();
    }
    if (q.t.loss_out && lane == 0 && loss_acc != 0.0) atomicAdd(q.t.loss_out, loss_acc);
}

// ---- pass 3: gradients ----
template <int MODEL>
__global__ void __launch_bounds__(SN_WARPS * 32) kge_shared_grad_kernel(const SharedNegParams q)
{
    constexpr int HALVES = (MODEL == KGE_TRANSE || MODEL == KGE_DISTMULT) ? 1 : 2;
    extern __shared__ __align__(16) float sn_smem[];
    float *const cand = sn_smem;
    float *const gc = sn_smem + SN_TJ * HALVES * SN_WK;  // the tile's candidate gradient rows of this window
    __shared__ int cid[SN_TJ];
    const Tile t = tile_of(q);
    if (t.i_begin >= t.i_end) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int eta = q.t.eta, kp = q.t.kp, ld = q.t.ld, nch = kp / 4, n_cb = (kp + SN_WK - 1) / SN_WK;
    const float scale = q.t.score_scale;
    tile_candidates(q, t, cid, false);
    __syncthreads();
    for (int cb = 0; cb < n_cb; ++cb) {
        for (int x = threadIdx.x; x < SN_TJ * HALVES * SN_WK / 4; x += blockDim.x) f4st(gc + 4 * x, f4zero());
        stage_window<HALVES>(q, cid, t.nt, cb, cand);
        __syncthreads();
        const int col = cb * 32 + lane, off = 4 * col;
        const bool live = col < nch;
#pragma unroll
        for (int u = 0; u < SN_PPW; ++u) {
            const long long i = t.i_begin + warp + SN_WARPS * u;
            if (i >= t.i_end) continue;
            const int s_id = q.t.triples[3 * i], p_id = q.t.triples[3 * i + 1], o_id = q.t.triples[3 * i + 2];
            PairOps<MODEL> S;
            S.load(q.t.ent + (size_t)s_id * ld, q.t.rel + (size_t)p_id * ld, q.t.ent + (size_t)o_id * ld, off, kp, live);
            const float g_l = lane < t.nt ? scale * q.sc[i * eta + t.j0 + lane] : 0.f;
            const unsigned side1 = __ballot_sync(0xffffffffu, lane < t.nt && q.keep[i * eta + t.j0 + lane] != 0);
            // each warp starts at its own candidate, so that the warps' shared-memory adds rarely meet on one row
            for (int n = 0, c = (4 * warp) % t.nt; n < t.nt; ++n, c = c + 1 == t.nt ? 0 : c + 1) {
                float4 r[2], d[2];
                read_row<MODEL>(cand, c, r);
                const float g = __shfl_sync(0xffffffffu, g_l, c);
                if ((side1 >> c) & 1u) S.template grad<1>(r, g, d);
                else S.template grad<0>(r, g, d);
                if (live) {
#pragma unroll
                    for (int h = 0; h < HALVES; ++h) {
                        float *dst = gc + (c * HALVES + h) * SN_WK + 4 * lane;
                        atomicAdd(dst + 0, d[h].x);
                        atomicAdd(dst + 1, d[h].y);
                        atomicAdd(dst + 2, d[h].z);
                        atomicAdd(dst + 3, d[h].w);
                    }
                }
            }
            if (live) {
                float4 gs[2], gp[2], go[2];
                S.finish(t.first ? scale * q.pos[i] : 0.f, q.t.inv_div, gs, gp, go);
                float *const gsr = q.t.grad_ent + (size_t)s_id * ld, *const gpr = q.t.grad_rel + (size_t)p_id * ld;
                float *const gor = q.t.grad_ent + (size_t)o_id * ld;
#pragma unroll
                for (int h = 0; h < HALVES; ++h) {
                    red_add_v4(gsr + h * kp + off, gs[h]);
                    red_add_v4(gor + h * kp + off, go[h]);
                    if (MODEL != KGE_ROTATE || h == 0) red_add_v4(gpr + h * kp + off, gp[h]);
                }
            }
        }
        __syncthreads();
        for (int x = threadIdx.x; x < t.nt * HALVES * 32; x += blockDim.x) {
            const int c = x & 31, h = (x >> 5) % HALVES, tt = (x >> 5) / HALVES;
            if (cb * 32 + c < nch)
                red_add_v4(q.t.grad_ent + (size_t)cid[tt] * ld + h * kp + 4 * (cb * 32 + c), f4ld(gc + (tt * HALVES + h) * SN_WK + 4 * c));
        }
        __syncthreads();
    }
}

template <int MODEL>
cudaError_t launch_shared_model(const SharedNegParams &q, int sm_count, cudaStream_t st)
{
    const long long grid = (long long)q.n_chunks * q.n_ps * q.n_jt;
    kge_shared_scores_kernel<MODEL><<<(unsigned)grid, SN_WARPS * 32, 0, st>>>(q);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    const long long want = (q.t.B + 7) / 8, cap = 16ll * sm_count;
    kge_shared_loss_kernel<<<(unsigned)(want < cap ? want : cap), 256, 0, st>>>(q);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    constexpr int HALVES = (MODEL == KGE_TRANSE || MODEL == KGE_DISTMULT) ? 1 : 2;
    return launch_with_smem(kge_shared_grad_kernel<MODEL>, dim3((unsigned)grid), SN_WARPS * 32,
                            2 * sizeof(float) * SN_TJ * HALVES * SN_WK, st, q);
}

}  // namespace

long long shared_negatives_grid(long long B, long long chunk, int eta, SharedNegParams *q)
{
    const long long n_chunks = (B + chunk - 1) / chunk, per = chunk < B ? chunk : B;
    const long long n_ps = (per + SN_PS - 1) / SN_PS, n_jt = (eta + SN_TJ - 1) / SN_TJ;
    if (q) { q->n_chunks = n_chunks; q->n_ps = n_ps; q->n_jt = (int)n_jt; }
    return n_chunks * n_ps * n_jt;
}

cudaError_t launch_shared_negatives(const SharedNegParams &q, int sm_count, cudaStream_t st)
{
    if (q.t.B == 0) return cudaSuccess;
    switch (q.t.model) {
    case KGE_TRANSE: return launch_shared_model<KGE_TRANSE>(q, sm_count, st);
    case KGE_DISTMULT: return launch_shared_model<KGE_DISTMULT>(q, sm_count, st);
    case KGE_COMPLEX: return launch_shared_model<KGE_COMPLEX>(q, sm_count, st);
    case KGE_HOLE: return launch_shared_model<KGE_HOLE>(q, sm_count, st);
    case KGE_ROTATE: return launch_shared_model<KGE_ROTATE>(q, sm_count, st);
    }
    return cudaErrorInvalidValue;
}

}  // namespace kge
