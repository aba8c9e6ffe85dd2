// kge_train.cu -- fused forward+backward of one training batch (sm_90a).
//
// Replaces, in ONE kernel: EmbeddingLookupLayer.call (layers/encoding/
// EmbeddingLookupLayer.py:307-342) for positives and corruptions,
// CorruptionGenerationLayerTrain.call (layers/corruption_generation/
// CorruptionGenerationLayerTrain.py:35-94), the five _compute_scores
// (layers/scoring/{TransE.py:37,DistMult.py:34,ComplEx.py:39,HolE.py:31,RotatE.py:62}),
// the five losses (loss_functions.py:286-308,360-382,442-464,540-574,630-654 via
// Loss.__call__ :185-225) and tape.gradient (optimizers.py:166).
//
// Work decomposition: one warp owns one positive and its eta corruptions at a
// time.  The warp's (3+G) embedding rows are gathered from HBM/L2 into its
// shared-memory slot by the copy engine (cp.async.bulk, one 1-D bulk copy per
// row, completion on a per-warp mbarrier); scores, loss and dL/dscore are
// computed from shared memory, which stays read-only after the gather; gradient
// float4s go straight from registers to the gradient tables with
// red.global.add.v4.f32.  (A copy-engine scatter -- cp.reduce.async.bulk of whole
// rows staged in shared memory -- and a two-warps-per-positive variant were both
// measured slower on cfg2 before the H100 port and removed.)  The reference re-gathers
// s,p,o for every corruption (3(1+eta) rows per positive); here each needed row
// moves once: (3+eta) rows in, (3+eta) gradient rows out = 2(3+eta)*ld*4 bytes
// per positive.
#include <math.h>

#include <type_traits>

#include "kge_train_common.cuh"

namespace kge {

// --------------------------------------------------------------------------
// Per-model scorers.  Each lane owns float4 chunks c = lane + 32*it (it < NIT) of every
// (padded) half-row; pad columns are zero in HBM and produce zero scores / gradients.
// All methods are warp-synchronous with no cross-lane traffic.  SIDE is a template
// argument (0 = subject replaced, 1 = object replaced): the caller partitions a
// positive's corruptions by side so the inner loops are branch-free, and feeds them in
// PAIRS (a, b) so two independent dependency chains are in flight.
//   prep(s,p,o)                      per-positive state; returns this lane's partial of f(s,p,o)
//   partial2<SIDE>(ra,rb,pa,pb)      partials of f for two corruptions with replaced rows ra, rb
//   grad2<SIDE>(...)                 RED g * df/dr for both rows, accumulate what the kept rows need
//   finish(...)                      RED the total gradient rows of s, p, o
// Unscaled f; HolE's 2/k factor is folded into g by the caller.  The formulas of DistMult, ComplEx / HolE and RotatE are
// the shared ones of kge_train_common.cuh (the fast paths use the same); TransE exists only here.
// --------------------------------------------------------------------------
template <int MODEL, int NIT>
struct Scorer;

// ---- DistMult: f = sum s*p*o (DistMult.py:48) -----------------------------
template <int NIT>
struct Scorer<KGE_DISTMULT, NIT> {
    float4 A[NIT], C[NIT], Ws[NIT], Wo[NIT];
    int lane, nch, cs = 32;  // cs: chunk stride = lanes cooperating on one positive
    // Lanes past the end of the window (c >= nch) carry ZERO query vectors (prep) and read the window's last chunk
    // instead of branching: their products are exact zeros, their W accumulators are never read, only their stores
    // are predicated.  The row loops are then branch-free, so the loads of all NIT iterations issue back to back.
    __device__ __forceinline__ int chunk(int it) const { return min(lane + cs * it, nch - 1); }
    __device__ __forceinline__ float prep(const float *s, const float *p, const float *o, int ln)
    {
        lane = ln;
        float4 acc = f4zero();
#pragma unroll
        for (int it = 0; it < NIT; ++it) {
            int c = lane + cs * it;
            float4 vs = f4zero(), vp = f4zero(), vo = f4zero();
            if (c < nch) { vs = f4ld(s + 4 * c); vp = f4ld(p + 4 * c); vo = f4ld(o + 4 * c); }
            A[it] = query_subj<1, 0>(vp, vp, vo, vo);
            C[it] = query_obj<1, 0>(vs, vs, vp, vp);
            Ws[it] = f4zero();
            Wo[it] = f4zero();
            acc = f4fma(vs, A[it], acc);
        }
        return f4hsum(acc);
    }
    template <int SIDE>
    __device__ __forceinline__ void partial2(const float *ra, const float *rb, float &pa, float &pb) const
    {
        float4 a = f4zero(), b = f4zero();
#pragma unroll
        for (int it = 0; it < NIT; ++it) {
            const int c = chunk(it);
            const float4 q = SIDE ? C[it] : A[it];
            a = f4fma(f4ld(ra + 4 * c), q, a);
            b = f4fma(f4ld(rb + 4 * c), q, b);
        }
        pa = f4hsum(a);
        pb = f4hsum(b);
    }
    static constexpr bool kQuad = true;  // has partial4: four corruptions of one side per call
    template <int SIDE>
    __device__ __forceinline__ void partial4(const float *r0, const float *r1, const float *r2, const float *r3, float &p0,
                                             float &p1, float &p2, float &p3) const
    {
        float4 a = f4zero(), b = f4zero(), c4 = f4zero(), d = f4zero();
#pragma unroll
        for (int it = 0; it < NIT; ++it) {
            const int c = chunk(it);
            const float4 q = SIDE ? C[it] : A[it];
            a = f4fma(f4ld(r0 + 4 * c), q, a);
            b = f4fma(f4ld(r1 + 4 * c), q, b);
            c4 = f4fma(f4ld(r2 + 4 * c), q, c4);
            d = f4fma(f4ld(r3 + 4 * c), q, d);
        }
        p0 = f4hsum(a); p1 = f4hsum(b); p2 = f4hsum(c4); p3 = f4hsum(d);
    }
    template <int SIDE>
    __device__ __forceinline__ void grad2(float *ra, float *rb, float *ga_row, float *gb_row, float ga, float gb,
                                          bool has_b)
    {
#pragma unroll
        for (int it = 0; it < NIT; ++it) {
            const int c = chunk(it);
            const bool live = lane + cs * it < nch;
            float4 va = f4ld(ra + 4 * c), vb = f4ld(rb + 4 * c);
            const float4 q = SIDE ? C[it] : A[it];
            float4 &W = SIDE ? Wo[it] : Ws[it];
            W = f4fma(ga, va, W);
            W = f4fma(gb, vb, W);
            if (live) red_add_v4(ga_row, 4 * c, ga * q);
            if (live && has_b) red_add_v4(gb_row, 4 * c, gb * q);
        }
    }
    __device__ __forceinline__ void finish(float *s, float *p, float *o, float *gs, float *gp, float *go, float gP,
                                           float)
    {
#pragma unroll
        for (int it = 0; it < NIT; ++it) {
            int c = lane + cs * it;
            if (c < nch) {
                float4 vs = f4ld(s + 4 * c), vp = f4ld(p + 4 * c), vo = f4ld(o + 4 * c);
                float4 U = f4fma(gP, vs, Ws[it]);  // everything that sat in the subject slot
                float4 X = f4fma(gP, vo, Wo[it]);  // everything that sat in the object slot
                red_add_v4(gs, 4 * c, query_subj<1, 0>(vp, vp, X, X));  // d/ds f(s,p,X)
                red_add_v4(go, 4 * c, query_obj<1, 0>(U, U, vp, vp));   // d/do f(U,p,o)
                red_add_v4(gp, 4 * c, trilinear_grad_p<1, 0>(vs, vs, vo, vo, U, U, Wo[it], Wo[it]));
            }
        }
    }
};

// ---- ComplEx / HolE (ComplEx.py:52-62; HolE.py:45 scales by 2/k) ----------
// f = sum s_re (p_re o_re + p_im o_im) + s_im (p_re o_im - p_im o_re); trilinear, so the
// kept-row gradients come from the weighted sums W of the replaced rows.
template <int NIT>
struct ComplexScorer {
    float4 A[NIT], Bv[NIT], C[NIT], D[NIT];          // subject-side / object-side query vectors
    float4 Wsr[NIT], Wsi[NIT], Wor[NIT], Woi[NIT];   // sum_j g_j r_j per side (re, im)
    int lane, nch, cs = 32, kp, hs;  // cs: chunk stride = lanes on one positive; kp: half stride in HBM rows, hs: half stride of the staged row window
    __device__ __forceinline__ int chunk(int it) const { return min(lane + cs * it, nch - 1); }  // see Scorer<KGE_DISTMULT>
    __device__ __forceinline__ float prep(const float *s, const float *p, const float *o, int ln)
    {
        lane = ln;
        float4 acc = f4zero();
#pragma unroll
        for (int it = 0; it < NIT; ++it) {
            int c = lane + cs * it;
            float4 sr = f4zero(), si = f4zero(), pr = f4zero(), pi = f4zero(), orr = f4zero(), oi = f4zero();
            if (c < nch) {
                sr = f4ld(s + 4 * c); si = f4ld(s + hs + 4 * c);
                pr = f4ld(p + 4 * c); pi = f4ld(p + hs + 4 * c);
                orr = f4ld(o + 4 * c); oi = f4ld(o + hs + 4 * c);
            }
            A[it] = query_subj<2, 0>(pr, pi, orr, oi); Bv[it] = query_subj<2, 1>(pr, pi, orr, oi);
            C[it] = query_obj<2, 0>(sr, si, pr, pi); D[it] = query_obj<2, 1>(sr, si, pr, pi);
            Wsr[it] = Wsi[it] = Wor[it] = Woi[it] = f4zero();
            acc = f4fma(sr, A[it], acc);
            acc = f4fma(si, Bv[it], acc);
        }
        return f4hsum(acc);
    }
    template <int SIDE>
    __device__ __forceinline__ void partial2(const float *ra, const float *rb, float &pa, float &pb) const
    {
        float4 a = f4zero(), b = f4zero();
#pragma unroll
        for (int it = 0; it < NIT; ++it) {
            const int c = chunk(it);
            const float4 qr = SIDE ? C[it] : A[it], qi = SIDE ? D[it] : Bv[it];
            a = f4fma(f4ld(ra + 4 * c), qr, a);
            b = f4fma(f4ld(rb + 4 * c), qr, b);
            a = f4fma(f4ld(ra + hs + 4 * c), qi, a);
            b = f4fma(f4ld(rb + hs + 4 * c), qi, b);
        }
        pa = f4hsum(a);
        pb = f4hsum(b);
    }
    static constexpr bool kQuad = true;
    template <int SIDE>
    __device__ __forceinline__ void partial4(const float *r0, const float *r1, const float *r2, const float *r3, float &p0,
                                             float &p1, float &p2, float &p3) const
    {
        float4 a = f4zero(), b = f4zero(), c4 = f4zero(), d = f4zero();
#pragma unroll
        for (int it = 0; it < NIT; ++it) {
            const int c = chunk(it);
            const float4 qr = SIDE ? C[it] : A[it], qi = SIDE ? D[it] : Bv[it];
            a = f4fma(f4ld(r0 + 4 * c), qr, a);
            b = f4fma(f4ld(r1 + 4 * c), qr, b);
            c4 = f4fma(f4ld(r2 + 4 * c), qr, c4);
            d = f4fma(f4ld(r3 + 4 * c), qr, d);
            a = f4fma(f4ld(r0 + hs + 4 * c), qi, a);
            b = f4fma(f4ld(r1 + hs + 4 * c), qi, b);
            c4 = f4fma(f4ld(r2 + hs + 4 * c), qi, c4);
            d = f4fma(f4ld(r3 + hs + 4 * c), qi, d);
        }
        p0 = f4hsum(a); p1 = f4hsum(b); p2 = f4hsum(c4); p3 = f4hsum(d);
    }
    template <int SIDE>
    __device__ __forceinline__ void grad2(float *ra, float *rb, float *ga_row, float *gb_row, float ga, float gb,
                                          bool has_b)
    {
#pragma unroll
        for (int it = 0; it < NIT; ++it) {
            const int c = chunk(it);
            const bool live = lane + cs * it < nch;
            float4 ar = f4ld(ra + 4 * c), ai = f4ld(ra + hs + 4 * c);
            float4 br = f4ld(rb + 4 * c), bi = f4ld(rb + hs + 4 * c);
            const float4 qr = SIDE ? C[it] : A[it], qi = SIDE ? D[it] : Bv[it];
            float4 &Wr = SIDE ? Wor[it] : Wsr[it];
            float4 &Wi = SIDE ? Woi[it] : Wsi[it];
            Wr = f4fma(ga, ar, Wr); Wi = f4fma(ga, ai, Wi);
            Wr = f4fma(gb, br, Wr); Wi = f4fma(gb, bi, Wi);
            if (live) {
                red_add_v4(ga_row, 4 * c, ga * qr);
                red_add_v4(ga_row, kp + 4 * c, ga * qi);
            }
            if (live && has_b) {
                red_add_v4(gb_row, 4 * c, gb * qr);
                red_add_v4(gb_row, kp + 4 * c, gb * qi);
            }
        }
    }
    __device__ __forceinline__ void finish(float *s, float *p, float *o, float *gs, float *gp, float *go, float gP,
                                           float)
    {
#pragma unroll
        for (int it = 0; it < NIT; ++it) {
            int c = lane + cs * it;
            if (c < nch) {
                float4 sr = f4ld(s + 4 * c), si = f4ld(s + hs + 4 * c);
                float4 pr = f4ld(p + 4 * c), pi = f4ld(p + hs + 4 * c);
                float4 orr = f4ld(o + 4 * c), oi = f4ld(o + hs + 4 * c);
                float4 Ur = f4fma(gP, sr, Wsr[it]), Ui = f4fma(gP, si, Wsi[it]);    // subject-slot mass
                float4 Xr = f4fma(gP, orr, Wor[it]), Xi = f4fma(gP, oi, Woi[it]);   // object-slot mass
                red_add_v4(gs, 4 * c, query_subj<2, 0>(pr, pi, Xr, Xi));  // d/ds f(s,p,X)
                red_add_v4(gs, kp + 4 * c, query_subj<2, 1>(pr, pi, Xr, Xi));
                red_add_v4(go, 4 * c, query_obj<2, 0>(Ur, Ui, pr, pi));   // d/do f(U,p,o)
                red_add_v4(go, kp + 4 * c, query_obj<2, 1>(Ur, Ui, pr, pi));
                red_add_v4(gp, 4 * c, trilinear_grad_p<2, 0>(sr, si, orr, oi, Ur, Ui, Wor[it], Woi[it]));
                red_add_v4(gp, kp + 4 * c, trilinear_grad_p<2, 1>(sr, si, orr, oi, Ur, Ui, Wor[it], Woi[it]));
            }
        }
    }
};
template <int NIT> struct Scorer<KGE_COMPLEX, NIT> : ComplexScorer<NIT> {};
template <int NIT> struct Scorer<KGE_HOLE, NIT> : ComplexScorer<NIT> {};

// ---- TransE: f = -sum |s+p-o| (TransE.py:51-53) ---------------------------
template <int NIT>
struct Scorer<KGE_TRANSE, NIT> {
    static constexpr bool kQuad = false;
    float4 Qs[NIT], Qo[NIT], Vs[NIT], Vo[NIT];  // p-o, s+p, sum g*sign per side
    int lane, nch, cs = 32;  // cs: chunk stride = lanes cooperating on one positive
    __device__ __forceinline__ float prep(const float *s, const float *p, const float *o, int ln)
    {
        lane = ln;
        float acc = 0.f;
#pragma unroll
        for (int it = 0; it < NIT; ++it) {
            int c = lane + cs * it;
            float4 vs = f4zero(), vp = f4zero(), vo = f4zero();
            if (c < nch) { vs = f4ld(s + 4 * c); vp = f4ld(p + 4 * c); vo = f4ld(o + 4 * c); }
            Qs[it] = vp - vo;
            Qo[it] = vs + vp;
            Vs[it] = Vo[it] = f4zero();
            acc -= f4abssum(Qo[it] - vo);
        }
        return acc;
    }
    template <int SIDE>
    __device__ __forceinline__ void partial2(const float *ra, const float *rb, float &pa, float &pb) const
    {
        float a = 0.f, b = 0.f;
#pragma unroll
        for (int it = 0; it < NIT; ++it) {
            int c = lane + cs * it;
            if (c < nch) {
                float4 va = f4ld(ra + 4 * c), vb = f4ld(rb + 4 * c);
                a -= f4abssum(SIDE ? (Qo[it] - va) : (va + Qs[it]));
                b -= f4abssum(SIDE ? (Qo[it] - vb) : (vb + Qs[it]));
            }
        }
        pa = a;
        pb = b;
    }
    template <int SIDE>
    __device__ __forceinline__ void grad2(float *ra, float *rb, float *ga_row, float *gb_row, float ga, float gb,
                                          bool has_b)
    {
#pragma unroll
        for (int it = 0; it < NIT; ++it) {
            int c = lane + cs * it;
            if (c < nch) {
                float4 va = f4ld(ra + 4 * c), vb = f4ld(rb + 4 * c);
                // SIDE 1: t = (s+p) - r, df/dr = +sign(t);  SIDE 0: t = r + (p-o), df/dr = -sign(t)
                float4 sa = ga * f4sgn(SIDE ? (Qo[it] - va) : (va + Qs[it]));
                float4 sb = gb * f4sgn(SIDE ? (Qo[it] - vb) : (vb + Qs[it]));
                float4 &V = SIDE ? Vo[it] : Vs[it];
                V = V + sa + sb;
                red_add_v4(ga_row, 4 * c, SIDE ? sa : f4neg(sa));
                if (has_b) red_add_v4(gb_row, 4 * c, SIDE ? sb : f4neg(sb));
            }
        }
    }
    __device__ __forceinline__ void finish(float *s, float *p, float *o, float *gs, float *gp, float *go, float gP,
                                           float)
    {
#pragma unroll
        for (int it = 0; it < NIT; ++it) {
            int c = lane + cs * it;
            if (c < nch) {
                float4 vo = f4ld(o + 4 * c);
                float4 Vp = gP * f4sgn(Qo[it] - vo);
                red_add_v4(gs, 4 * c, f4neg(Vp + Vo[it]));
                red_add_v4(gp, 4 * c, f4neg(Vp + Vs[it] + Vo[it]));
                red_add_v4(go, 4 * c, Vp + Vs[it]);
            }
        }
    }
};

// ---- RotatE (kge_train_common.cuh: rot_*) ----------------------------------
// The relation row handed to this kernel is the per-step rotation table row [cos(phi) | sin(phi)], phi = theta/div
// (kge_rotation_table_kernel).  Lanes past the end of the window are masked arithmetically (they read the window's
// last chunk; only their stores are predicated) so the row loops carry no divergence bookkeeping.
template <int NIT>
struct Scorer<KGE_ROTATE, NIT> {
    static constexpr bool kQuad = false;
    float4 C[NIT], Sn[NIT], Or_[NIT], Oi[NIT], Yr[NIT], Yi[NIT];
    float4 Zor[NIT], Zoi[NIT], Zsr[NIT], Zsi[NIT], Aphi[NIT];
    float nlive[NIT];  // -1 for a lane that owns a chunk of this window, 0 past its end
    int lane, nch, cs = 32, kp, hs;  // cs: chunk stride = lanes on one positive; kp: half stride in HBM rows, hs: half stride of the staged row window
    __device__ __forceinline__ int chunk(int it) const { return min(lane + cs * it, nch - 1); }
    __device__ __forceinline__ float prep(const float *s, const float *p, const float *o, int ln)
    {
        lane = ln;
        float acc = 0.f;
#pragma unroll
        for (int it = 0; it < NIT; ++it) {
            const int c = lane + cs * it;
            float4 sr = f4zero(), si = f4zero();
            C[it] = Sn[it] = Or_[it] = Oi[it] = f4zero();
            nlive[it] = 0.f;
            if (c < nch) {
                sr = f4ld(s + 4 * c); si = f4ld(s + hs + 4 * c);
                C[it] = f4ld(p + 4 * c); Sn[it] = f4ld(p + hs + 4 * c);
                Or_[it] = f4ld(o + 4 * c); Oi[it] = f4ld(o + hs + 4 * c);
                nlive[it] = -1.f;
            }
            Yr[it] = rot_rotate<0>(sr, si, C[it], Sn[it]);
            Yi[it] = rot_rotate<1>(sr, si, C[it], Sn[it]);
            Zor[it] = Zoi[it] = Zsr[it] = Zsi[it] = Aphi[it] = f4zero();
            acc = fmaf(rot_modsum(Yr[it] - Or_[it], Yi[it] - Oi[it]), nlive[it], acc);
        }
        return acc;
    }
    template <int SIDE>
    __device__ __forceinline__ void partial2(const float *ra, const float *rb, float &pa, float &pb) const
    {
        float a = 0.f, b = 0.f;
#pragma unroll
        for (int it = 0; it < NIT; ++it) {
            const int c = chunk(it);
            const float4 ar = f4ld(ra + 4 * c), ai = f4ld(ra + hs + 4 * c);
            const float4 br = f4ld(rb + 4 * c), bi = f4ld(rb + hs + 4 * c);
            if (SIDE) {  // y - r
                a = fmaf(rot_modsum(Yr[it] - ar, Yi[it] - ai), nlive[it], a);
                b = fmaf(rot_modsum(Yr[it] - br, Yi[it] - bi), nlive[it], b);
            } else {
                const float4 e0 = rot_residual_subj<0>(ar, ai, C[it], Sn[it], Or_[it], Oi[it]);
                const float4 e1 = rot_residual_subj<1>(ar, ai, C[it], Sn[it], Or_[it], Oi[it]);
                const float4 e2 = rot_residual_subj<0>(br, bi, C[it], Sn[it], Or_[it], Oi[it]);
                const float4 e3 = rot_residual_subj<1>(br, bi, C[it], Sn[it], Or_[it], Oi[it]);
                a = fmaf(rot_modsum(e0, e1), nlive[it], a);
                b = fmaf(rot_modsum(e2, e3), nlive[it], b);
            }
        }
        pa = a;
        pb = b;
    }
    template <int SIDE>
    __device__ __forceinline__ void grad1(float *r, float *grow, float g, int it, int c, bool emit)
    {
        const float4 rr = f4ld(r + 4 * c), ri = f4ld(r + hs + 4 * c);
        float4 a, b;
        if (SIDE) {  // residual = y(s) - r ; df/dr = +(a,b)
            rot_unit(Yr[it] - rr, Yi[it] - ri, g, a, b);
            Zor[it] = Zor[it] + a; Zoi[it] = Zoi[it] + b;
            if (emit) { red_add_v4(grow, 4 * c, a); red_add_v4(grow, kp + 4 * c, b); }
        } else {  // residual = R(phi) r - o ; df/dr = -R(-phi)(a,b)
            const float4 yr = rot_rotate<0>(rr, ri, C[it], Sn[it]), yi = rot_rotate<1>(rr, ri, C[it], Sn[it]);  // R(phi) r
            rot_unit(yr - Or_[it], yi - Oi[it], g, a, b);
            Zsr[it] = Zsr[it] + a; Zsi[it] = Zsi[it] + b;
            Aphi[it] = rot_dphi(a, b, yr, yi, Aphi[it]);
            if (emit) {
                red_add_v4(grow, 4 * c, rot_back<0>(a, b, C[it], Sn[it]));
                red_add_v4(grow, kp + 4 * c, rot_back<1>(a, b, C[it], Sn[it]));
            }
        }
    }
    template <int SIDE>
    __device__ __forceinline__ void grad2(float *ra, float *rb, float *ga_row, float *gb_row, float ga, float gb,
                                          bool has_b)
    {
#pragma unroll
        for (int it = 0; it < NIT; ++it) {
            const int c = chunk(it);
            const bool live = lane + cs * it < nch;  // dead lanes run the arithmetic on the last chunk; their accumulators are never read
            grad1<SIDE>(ra, ga_row, ga, it, c, live);
            grad1<SIDE>(rb, gb_row, gb, it, c, live && has_b);  // gb == 0 when !has_b: contributes nothing
        }
    }
    // p row receives d/dtheta = (1/div) d/dphi in its first half, zeros in the second
    // (the second half of a RotatE relation row is allocated but unused, RotatE.py:76).
    __device__ __forceinline__ void finish(float *s, float *p, float *o, float *gs, float *gp, float *go, float gP,
                                           float inv_div)
    {
#pragma unroll
        for (int it = 0; it < NIT; ++it) {
            int c = lane + cs * it;
            if (c < nch) {
                float4 a, b;
                rot_unit(Yr[it] - Or_[it], Yi[it] - Oi[it], gP, a, b);
                const float4 Zr = a + Zor[it], Zi = b + Zoi[it];  // everything with y = R(phi) s
                red_add_v4(gs, 4 * c, rot_back<0>(Zr, Zi, C[it], Sn[it]));
                red_add_v4(gs, kp + 4 * c, rot_back<1>(Zr, Zi, C[it], Sn[it]));
                red_add_v4(go, 4 * c, a + Zsr[it]);
                red_add_v4(go, kp + 4 * c, b + Zsi[it]);
                red_add_v4(gp, 4 * c, inv_div * rot_dphi(Zr, Zi, Yr[it], Yi[it], Aphi[it]));
            }
        }
    }
};

// --------------------------------------------------------------------------
// the kernel
// --------------------------------------------------------------------------

// Visit the resident corruptions [0, gs) of one group, partitioned by side and two at a
// time: f(side_tag, slot_a, slot_b, has_b).  nside[] holds keep_subj (1 = object replaced).
template <class F0, class F1>
__device__ __forceinline__ void for_each_pair_by_side(const int *nside, int gs, int lane, F0 f0, F1 f1)
{
    for (int base = 0; base < gs; base += 32) {
        const int jl = base + lane;
        const int sd = (jl < gs) ? nside[jl] : -1;
#pragma unroll
        for (int side = 0; side < 2; ++side) {
            unsigned m = __ballot_sync(0xffffffffu, sd == side);
            while (m) {
                const int a = base + __ffs(m) - 1;
                m &= m - 1;
                int b = a;
                const bool has_b = m != 0;
                if (has_b) { b = base + __ffs(m) - 1; m &= m - 1; }
                if (side == 0) f0(a, b, has_b); else f1(a, b, has_b);
            }
        }
    }
}

// Shared-memory slot of one warp: (3+G) row WINDOWS.  A window is the [cb*wk, cb*wk+wk) column
// slice of each half of a row (wk = min(kp, 128*NIT) floats), so one positive's working set is
// bounded in registers (NIT float4 per lane per vector) and in shared memory whatever k and eta
// are: columns are processed window by window (scores add up over windows), negatives group by
// group.  With one window and one group (the common case: cfg2/cfg3) every row is gathered once
// and stays resident for the gradient pass.
// Row-sharded tables (SURVEY.md 8e, cfg4/cfg5): entity id e lives on rank e / rows_per_shard at local row
// e % rows_per_shard; every shard is peer-mapped, so the SAME bulk gathers and red.v4 scatters reach
// remote shards through NVLink -- the row all-to-all is fused into the kernel.
__device__ __forceinline__ const float *ent_row(const TrainParams &p, int id)
{
    if (p.shard_world <= 1) return p.ent + (size_t)id * p.ld;
    const int q = id / p.rows_per_shard;
    return p.ent_shard[q] + (size_t)(id - q * p.rows_per_shard) * p.ld;
}
__device__ __forceinline__ void stamp_ent_row(const TrainParams &p, int id)
{
    if (p.shard_world <= 1) { p.stamp_ent[id] = p.stamp; return; }
    const int q = id / p.rows_per_shard;
    p.stamp_ent_shard[q][id - q * p.rows_per_shard] = p.stamp;
}
__device__ __forceinline__ float *gent_row(const TrainParams &p, int id)
{
    if (p.shard_world <= 1) return p.grad_ent + (size_t)id * p.ld;
    const int q = id / p.rows_per_shard;
    return p.grad_ent_shard[q] + (size_t)(id - q * p.rows_per_shard) * p.ld;
}

// RESIDENT = one window and one group (decided on the host): the window/group machinery folds away.
template <int MODEL, int NIT, bool RESIDENT>
__global__ void __launch_bounds__(KGE_TRAIN_THREADS(MODEL, NIT)) kge_train_kernel(const TrainParams p)
{
    constexpr int HALVES = (MODEL == KGE_TRANSE || MODEL == KGE_DISTMULT) ? 1 : 2;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    unsigned char *region = smem_raw + (size_t)warp * p.region_bytes;
    float *rows = reinterpret_cast<float *>(region);  // (3+G) windows of lw floats
    float *sc = reinterpret_cast<float *>(region + p.rows_bytes);
    int *nid = reinterpret_cast<int *>(sc + p.eta_pad);
    int *nside = nid + p.eta_pad;   // scratch while the corruptions are being sorted
    int *jorig = nside + p.eta_pad; // sorted slot -> index j of the corruption in the reference's tile order
    uint64_t *bar = reinterpret_cast<uint64_t *>(jorig + p.eta_pad);

    if (lane == 0) { mbar_init(bar, 1); mbar_init(bar + 1, 1); }
    fence_mbar_init();
    fence_proxy_async_smem();
    __syncthreads();

    const int ld = p.ld, kp = p.kp, eta = p.eta, G = RESIDENT ? p.eta : p.G;
    const int wk = RESIDENT ? p.kp : p.wk;     // window floats per half
    const int lw = p.slot_floats;              // slot stride (>= HALVES*wk)
    const int n_cb = RESIDENT ? 1 : p.n_cb;    // column windows per row
    const int n_groups = RESIDENT ? 1 : (eta + G - 1) / G;
    // (making these loop invariants opaque to the front end, as kge_train_res.cu does, was measured to change nothing here before the H100 port)
    constexpr bool resident = RESIDENT;
    // slot: s, p, o windows, then group buffer 0 and (non-resident, p.nbuf == 2) group buffer 1: the next group is
    // gathered while the current one is being processed, which hides the gather latency inside the warp (NVLink
    // latency when the table is row-sharded over GPUs).  With p.nbuf == 1 the next group is requested when the
    // current one has been consumed and the latency is hidden by the OTHER warps of the SM instead: half the
    // shared memory per warp, so more warps (kge_create picks per shape).
    const bool dbuf = !RESIDENT && p.nbuf == 2;
    float *srow = rows, *prow = rows + lw, *orow = rows + 2 * lw;
    auto nbuf = [&](int b) { return rows + (size_t)(3 + b * G) * lw; };
    const float scale = p.score_scale;  // HolE 2/k, else 1
    uint32_t phase0 = 0u, phase1 = 0u;
    double loss_acc = 0.0;

    const long long n_warps = (long long)gridDim.x * (blockDim.x >> 5);
    float next_draw = 0.f;  // lane 0: this warp's draw from the positive counter (kge_train_common.cuh: dynamic assignment)
    for (long long i = (long long)blockIdx.x * (blockDim.x >> 5) + warp; i < p.B;
         i = p.sched ? n_warps + (long long)(unsigned)__shfl_sync(0xffffffffu, next_draw, 0) : i + n_warps) {
        if (p.sched && lane == 0) next_draw = sched_draw(p.sched);  // consumed by the loop increment, a whole positive later
        const int s_id = p.triples[3 * i], p_id = p.triples[3 * i + 1], o_id = p.triples[3 * i + 2];
        // ---- corruptions of this positive (A3), SORTED BY SIDE as they are drawn ----
        // Slot t of the warp's arrays (nid, sc, the gathered rows, the stash) holds corruption jorig[t]; slots [0, n0)
        // replaced the subject, slots [n0, eta) the object.  Both passes then walk two plain index ranges with the side
        // as a template argument -- no ballot / find-first-set bookkeeping per pair of corruptions.
        int n0 = 0;
        for (int base = 0; base < eta; base += 32) {
            const int j = base + lane;
            int keep = 1, repl = 0;
            if (j < eta) {
                corruption_of(p, (unsigned long long)j * (unsigned long long)p.B + (unsigned long long)i, keep, repl);
                nside[j] = keep;  // keep_subj = 1 -> object replaced -> side 1
                sc[j] = __int_as_float(repl);
                if (p.stamp_ent && p.mode != KGE_STEP_FORWARD_ONLY) stamp_ent_row(p, repl);  // lazy optimizer: row touched
            }
            n0 += __popc(__ballot_sync(0xffffffffu, j < eta && keep == 0));
        }
        __syncwarp();
        {
            int c0 = 0, c1 = n0;
            const unsigned lt = (1u << lane) - 1u;
            for (int base = 0; base < eta; base += 32) {
                const int j = base + lane;
                const int keep = (j < eta) ? nside[j] : -1;
                const unsigned m0 = __ballot_sync(0xffffffffu, keep == 0), m1 = __ballot_sync(0xffffffffu, keep == 1);
                if (j < eta) {
                    const int t = keep ? c1 + __popc(m1 & lt) : c0 + __popc(m0 & lt);
                    nid[t] = __float_as_int(sc[j]);
                    jorig[t] = j;
                }
                c0 += __popc(m0);
                c1 += __popc(m1);
            }
        }
        __syncwarp();
        if (!resident)
            for (int j = lane; j < eta; j += 32) sc[j] = 0.f;
        if (p.stamp_ent && p.mode != KGE_STEP_FORWARD_ONLY) {
            if (lane == 0) stamp_ent_row(p, s_id);
            if (lane == 1) stamp_ent_row(p, o_id);
            if (lane == 2 && p.stamp_rel) p.stamp_rel[p_id] = p.stamp;
        }
        __syncwarp();
        float *const gs_row = gent_row(p, s_id), *const gp_row = p.grad_rel + (size_t)p_id * ld, *const go_row = gent_row(p, o_id);

        // issue the gather of (optionally) the s,p,o windows and of group [j0, j0+gsz) into buffer `buf`:
        // one 1-D bulk copy per row window, completion counted on the buffer's mbarrier
        // from_stash: the gradient pass of a row-sharded run re-reads the replaced rows from the LOCAL stash the score
        // pass filled, instead of pulling them through NVLink a second time
        auto issue = [&](int buf, int cb, bool with_spo, int j0, int gsz, bool from_stash = false) {
            const int wch_t = min(wk, kp - cb * wk);  // floats of this window per half
            const uint32_t bytes = (n_cb == 1) ? (uint32_t)ld * 4u : (uint32_t)wch_t * 4u;
            const int copies = (n_cb == 1) ? 1 : HALVES;
            const int nspo = with_spo ? 3 : 0, total = (nspo + gsz) * copies;
            if (lane == 0) mbar_arrive_expect_tx(bar + buf, (uint32_t)total * bytes);
            __syncwarp();
            float *const gb = nbuf(buf);
            for (int r = lane; r < total; r += 32) {
                const int row = (copies == 1) ? r : r / HALVES, h = (copies == 1) ? 0 : r - row * HALVES;
                const float *src;
                float *dst;
                if (row < nspo) {
                    src = row == 0 ? ent_row(p, s_id) : row == 1 ? p.rel + (size_t)p_id * ld : ent_row(p, o_id);
                    dst = rows + (size_t)row * lw;
                } else {
                    src = from_stash ? p.stash + ((size_t)i * eta + (j0 + row - nspo)) * ld : ent_row(p, nid[j0 + row - nspo]);
                    dst = gb + (size_t)(row - nspo) * lw;
                }
                bulk_load(dst + h * wk, src + h * kp + cb * wk, bytes, bar + buf);
            }
        };
        auto wait = [&](int buf) {
            if (buf) { mbar_wait(bar + 1, phase1); phase1 ^= 1u; }
            else { mbar_wait(bar, phase0); phase0 ^= 1u; }
        };
        // copy the group rows just gathered (possibly from a peer GPU) into this rank's stash
        auto stash_rows = [&](int buf, int cb, int j0, int gsz) {
            const int wch_t = min(wk, kp - cb * wk);
            const uint32_t bytes = (n_cb == 1) ? (uint32_t)ld * 4u : (uint32_t)wch_t * 4u;
            const int copies = (n_cb == 1) ? 1 : HALVES;
            float *const gb = nbuf(buf);
            for (int r = lane; r < gsz * copies; r += 32) {
                const int row = (copies == 1) ? r : r / HALVES, h = (copies == 1) ? 0 : r - row * HALVES;
                bulk_store(p.stash + ((size_t)i * eta + (j0 + row)) * ld + h * kp + cb * wk, gb + (size_t)row * lw + h * wk, bytes);
            }
            bulk_commit();
        };
        const bool use_stash = !RESIDENT && p.stash != nullptr;
        Scorer<MODEL, NIT> S;
        if constexpr (HALVES == 2) { S.kp = kp; S.hs = wk; }
        float P = 0.f;

        // ---- pass A: scores, window by window, group by group, next group prefetched (A2 + A4) ----
        for (int cb = 0; cb < n_cb; ++cb) {
            S.nch = min(wk, kp - cb * wk) / 4;
            if (use_stash) bulk_wait_read_all();
            __syncwarp();
            issue(0, cb, true, 0, min(G, eta));
            for (int g = 0; g < n_groups; ++g) {
                const int buf = dbuf ? (g & 1) : 0, j0 = g * G, gsz = min(G, eta - j0);
                if (dbuf && g + 1 < n_groups) {
                    if (use_stash) { bulk_wait_read_all(); __syncwarp(); }  // the stash store of group g-1 has read buf^1
                    issue(buf ^ 1, cb, false, j0 + G, min(G, eta - j0 - G));
                }
                wait(buf);
                if (use_stash) stash_rows(buf, cb, j0, gsz);
                if (g == 0) P += warp_sum(S.prep(srow, prow, orow, lane));
                float *const nrows = nbuf(buf);
                // reduce the two partials over the warp (lower half-warp ends up with a's sum, upper with b's) and store
                auto store = [&](int a, int b, bool has_b, float pa, float pb) {
                    const float v = warp_sum2t(pa, pb, lane);
                    if ((lane & 15) == 0 && (lane == 0 || has_b)) {
                        const int t = j0 + (lane ? b : a);
                        if (resident) sc[t] = v; else sc[t] += v;
                    }
                };
                // slots [j0, j0+gsz) of this group: the part below n0 replaced the subject, the rest the object
                const int e0 = min(n0, j0 + gsz), b1 = max(n0, j0);
                if constexpr (Scorer<MODEL, NIT>::kQuad) {
                    // four corruptions per trip; slots past the end of the range alias the last valid one and are dropped
                    auto quad = [&](int t, int end, auto side_tag) {
                        constexpr int SIDE = decltype(side_tag)::value;
                        const int last = end - 1 - j0, a0 = t - j0;
                        const float *r0 = nrows + (size_t)a0 * lw, *r1 = nrows + (size_t)min(a0 + 1, last) * lw;
                        const float *r2 = nrows + (size_t)min(a0 + 2, last) * lw, *r3 = nrows + (size_t)min(a0 + 3, last) * lw;
                        float v0, v1, v2, v3;
                        S.template partial4<SIDE>(r0, r1, r2, r3, v0, v1, v2, v3);
                        const float v = warp_sum4t(v0, v1, v2, v3, lane);
                        const int q = lane >> 3;
                        if ((lane & 7) == 0 && t + q < end) {
                            if (resident) sc[t + q] = v; else sc[t + q] += v;
                        }
                    };
                    // a tail of one or two corruptions takes the cheaper two-at-a-time path
                    auto tail = [&](int t, int end, auto side_tag) {
                        constexpr int SIDE = decltype(side_tag)::value;
                        const int a = t - j0;
                        const bool has_b = t + 1 < end;
                        const int b = has_b ? a + 1 : a;
                        float pa, pb;
                        S.template partial2<SIDE>(nrows + (size_t)a * lw, nrows + (size_t)b * lw, pa, pb);
                        store(a, b, has_b, pa, pb);
                    };
                    auto side_range = [&](int lo, int hi, auto side_tag) {
                        int t = lo;
                        for (; hi - t >= 3; t += 4) quad(t, hi, side_tag);
                        if (t < hi) tail(t, hi, side_tag);
                    };
                    side_range(j0, e0, std::integral_constant<int, 0>{});
                    side_range(b1, j0 + gsz, std::integral_constant<int, 1>{});
                } else {
                for (int t = j0; t < e0; t += 2) {
                    const int a = t - j0;
                    const bool has_b = t + 1 < e0;
                    const int b = has_b ? a + 1 : a;
                    float pa, pb;
                    S.template partial2<0>(nrows + (size_t)a * lw, nrows + (size_t)b * lw, pa, pb);
                    store(a, b, has_b, pa, pb);
                }
                for (int t = b1; t < j0 + gsz; t += 2) {
                    const int a = t - j0;
                    const bool has_b = t + 1 < j0 + gsz;
                    const int b = has_b ? a + 1 : a;
                    float pa, pb;
                    S.template partial2<1>(nrows + (size_t)a * lw, nrows + (size_t)b * lw, pa, pb);
                    store(a, b, has_b, pa, pb);
                }
                }
                __syncwarp();
                if (!dbuf && g + 1 < n_groups) {  // single buffer: every lane is done with this group, fetch the next one over it
                    if (use_stash) { bulk_wait_read_all(); __syncwarp(); }  // ... and so is the stash store
                    issue(0, cb, false, j0 + G, min(G, eta - j0 - G));
                }
            }
        }

        // ---- loss and dL/dscore (A5) ----
        float dP;
        if (p.mode != KGE_STEP_BACKWARD_EXT) {
            if (scale != 1.f)
                for (int j = lane; j < eta; j += 32) sc[j] *= scale;
            __syncwarp();
            if (p.scores_neg)
                for (int t = lane; t < eta; t += 32) p.scores_neg[(size_t)jorig[t] * p.B + i] = sc[t];
            if (p.scores_pos && lane == 0) p.scores_pos[i] = scale * P;
            if (p.mode == KGE_STEP_FORWARD_ONLY) { __syncwarp(); continue; }
            float li = loss_and_dscores(p, scale * P, sc, lane, &dP);
            if (lane == 0) loss_acc += (double)li;
        } else {
            for (int t = lane; t < eta; t += 32) sc[t] = p.dneg[(size_t)jorig[t] * p.B + i];
            dP = p.dpos[i];
        }
        __syncwarp();

        if (use_stash) { bulk_wait_all(); __syncwarp(); }  // stash rows are in HBM before the gradient pass reads them

        // ---- pass B: gradients, last window / last group first (they are still resident) ----
        for (int cb = n_cb - 1; cb >= 0; --cb) {
            S.nch = min(wk, kp - cb * wk) / 4;
            const int gofs = cb * wk;  // column offset of this window inside a gradient row
            for (int g = n_groups - 1; g >= 0; --g) {
                const int buf = dbuf ? (g & 1) : 0, j0 = g * G, gsz = min(G, eta - j0);
                const bool top = (g == n_groups - 1);
                const bool still_there = (cb == n_cb - 1 && top);  // left in place by pass A
                if (top && !still_there) {  // first visit of this window: s, p, o come along, state is rebuilt
                    __syncwarp();
                    issue(buf, cb, true, j0, gsz, use_stash);
                }
                if (dbuf && g > 0) {  // prefetch the next (lower) group into the other buffer
                    __syncwarp();
                    issue(buf ^ 1, cb, false, j0 - G, G, use_stash);
                }
                if (!still_there) wait(buf);
                if (top && !still_there) (void)S.prep(srow, prow, orow, lane);
                float *const nrows = nbuf(buf);
                const int e0 = min(n0, j0 + gsz), b1 = max(n0, j0);
                for (int t = j0; t < e0; t += 2) {
                    const int a = t - j0;
                    const bool has_b = t + 1 < e0;
                    const int b = has_b ? a + 1 : a;
                    S.template grad2<0>(nrows + (size_t)a * lw, nrows + (size_t)b * lw, gent_row(p, nid[j0 + a]) + gofs,
                                        gent_row(p, nid[j0 + b]) + gofs, scale * sc[j0 + a],
                                        has_b ? scale * sc[j0 + b] : 0.f, has_b);
                }
                for (int t = b1; t < j0 + gsz; t += 2) {
                    const int a = t - j0;
                    const bool has_b = t + 1 < j0 + gsz;
                    const int b = has_b ? a + 1 : a;
                    S.template grad2<1>(nrows + (size_t)a * lw, nrows + (size_t)b * lw, gent_row(p, nid[j0 + a]) + gofs,
                                        gent_row(p, nid[j0 + b]) + gofs, scale * sc[j0 + a],
                                        has_b ? scale * sc[j0 + b] : 0.f, has_b);
                }
                __syncwarp();
                if (!dbuf && g > 0) issue(0, cb, false, j0 - G, G, use_stash);  // single buffer: the next (lower) group over this one
            }
            S.finish(srow, prow, orow, gs_row + gofs, gp_row + gofs, go_row + gofs, scale * dP, p.inv_div);
        }
        __syncwarp();
    }
    sched_retire(p.sched, n_warps, lane);
    if (p.loss_out && p.mode == KGE_STEP_FUSED && lane == 0 && loss_acc != 0.0) atomicAdd(p.loss_out, loss_acc);
}

// --------------------------------------------------------------------------
// RotatE rotation table: rot[r] = [cos(theta/div) | sin(theta/div)] (RotatE.py:96-98),
// canonical sin/cos so that training, predict and ranking agree bit for bit.
// --------------------------------------------------------------------------
__global__ void kge_rotation_table_kernel(const float *__restrict__ rel, float *__restrict__ rot, long long n_rel,
                                          int kp, int ld, float div)
{
    long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n_rel * kp) return;
    long long r = idx / kp;
    int d = (int)(idx - r * kp);
    float s, c;
    kge_sincosf(__fdiv_rn(rel[r * ld + d], div), &s, &c);
    rot[r * ld + d] = c;
    rot[r * ld + kp + d] = s;
}

// --------------------------------------------------------------------------
// materialise the Philox corruption stream (inspection / parity only)
// --------------------------------------------------------------------------
__global__ void kge_corruptions_kernel(const int32_t *__restrict__ triples, long long B, int eta,
                                       unsigned long long seed, unsigned long long step, unsigned n_ent,
                                       int32_t *__restrict__ out)
{
    long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= B * eta) return;
    long long i = r % B;
    int keep, repl;
    draw_corruption(seed, step, (unsigned long long)r, n_ent, &keep, &repl);
    out[3 * r + 0] = keep ? triples[3 * i + 0] : repl;
    out[3 * r + 1] = triples[3 * i + 1];
    out[3 * r + 2] = keep ? repl : triples[3 * i + 2];
}

// --------------------------------------------------------------------------
// host launchers
// --------------------------------------------------------------------------
template <int MODEL, int NIT>
static cudaError_t launch_train_nit(const TrainParams &p, const TrainSlot &slot, int sm_count, cudaStream_t st)
{
    return launch_persistent(p.resident ? kge_train_kernel<MODEL, NIT, true> : kge_train_kernel<MODEL, NIT, false>, p, slot,
                             sm_count, st);
}

template <int MODEL>
static cudaError_t launch_train_model(const TrainParams &p, int nit, const TrainSlot &slot, int sm_count, cudaStream_t st)
{
    switch (nit) {
    case 1: return launch_train_nit<MODEL, 1>(p, slot, sm_count, st);
    case 2: return launch_train_nit<MODEL, 2>(p, slot, sm_count, st);
    case 4: return launch_train_nit<MODEL, 4>(p, slot, sm_count, st);
    }
    return cudaErrorInvalidValue;
}

cudaError_t launch_train(const TrainParams &p, int nit, const TrainSlot &slot, int sm_count, cudaStream_t st)
{
    switch (p.model) {
    case KGE_TRANSE: return launch_train_model<KGE_TRANSE>(p, nit, slot, sm_count, st);
    case KGE_DISTMULT: return launch_train_model<KGE_DISTMULT>(p, nit, slot, sm_count, st);
    case KGE_COMPLEX: return launch_train_model<KGE_COMPLEX>(p, nit, slot, sm_count, st);
    case KGE_HOLE: return launch_train_model<KGE_HOLE>(p, nit, slot, sm_count, st);
    case KGE_ROTATE: return launch_train_model<KGE_ROTATE>(p, nit, slot, sm_count, st);
    }
    return cudaErrorInvalidValue;
}

cudaError_t launch_rotation_table(const float *rel, float *rot, long long n_rel, int kp, int ld, float div,
                                  cudaStream_t st)
{
    long long n = n_rel * kp;
    if (n == 0) return cudaSuccess;
    kge_rotation_table_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(rel, rot, n_rel, kp, ld, div);
    return cudaGetLastError();
}

cudaError_t launch_corruptions(const int32_t *triples, long long B, int eta, unsigned long long seed,
                               unsigned long long step, unsigned n_ent, int32_t *out, cudaStream_t st)
{
    long long n = B * eta;
    if (n == 0) return cudaSuccess;
    kge_corruptions_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(triples, B, eta, seed, step, n_ent, out);
    return cudaGetLastError();
}

}  // namespace kge
