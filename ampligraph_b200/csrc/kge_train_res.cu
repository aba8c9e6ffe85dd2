// kge_train_res.cu -- the RESIDENT TRILINEAR fast path of the fused training step (sm_90a).
//
// Same contract as kge_train_kernel (kge_train.cu; reference: train_step ScoringBasedEmbeddingModel.py:370-429 ->
// EmbeddingLookupLayer.call, CorruptionGenerationLayerTrain.call, DistMult/ComplEx/HolE _compute_scores, the five
// losses, tape.gradient), specialised for the shape the headline workload has: DistMult / ComplEx / HolE, every row of
// a positive resident in the warp's shared-memory slot (one column window, one group), eta <= 32 (one corruption per
// lane), a single (not row-sharded) table.  What the specialisation buys (in the general kernel fewer than half the
// instructions of the gradient loop are loads / FMAs / REDs): all shared-memory traffic goes through explicit 32-bit shared addresses (one IADD per
// 128-bit load instead of 64-bit generic pointer arithmetic re-derived every trip), gradient rows are addressed as
// one 64-bit base per row plus the lane's byte offset, the shard/window/group machinery does not exist, and the
// corruption sort is one ballot pair.  The per-element arithmetic is the general kernel's: both form the query vectors
// and the kept rows' gradients with query_subj / query_obj / trilinear_grad_p (kge_train_common.cuh), so both
// produce the same scores; gradients differ only in the order of the fp32 atomics.
#include "kge_train_common.cuh"

namespace kge {

#ifndef KGE_HOT
#define KGE_HOT 1  // entities whose subject/object gradient rows are privatised per warp (1 or 2; 2 measured no faster on cfg2 and slower on uniform triples before the H100 port)
#endif

// RED of one chunk of a replaced entity's gradient row.  -DKGE_PROFILE_NOREPLRED builds a profiling variant that drops
// only these (the s / p / o rows keep theirs): how much of the kernel the uniformly scattered replaced-row REDs cost.
__device__ __forceinline__ void red_repl_v4(float *g, float4 v)
{
#ifdef KGE_PROFILE_NOREPLRED
    if (v.x != 1.2345e38f) return;  // profiling build: the RED is dropped, v stays live
#endif
    red_add_v4(g, v);
}

// ---- the kernel ----------------------------------------------------------------------------------------------------------
// HALVES = 1: DistMult (f = sum s p o, DistMult.py:48); HALVES = 2: ComplEx / HolE (ComplEx.py:52-62; HolE.py:45 scales by
// 2/k, folded into the gradient scalars).  Lane l owns float4 chunks c = l + 32*it (it < NIT) of every half-row; lanes past
// the end of the row read its last chunk with zero query vectors (exact zeros in every sum) and never store.
// Shared-memory slot of a warp (kge_create: the resident trilinear TrainSlot, p.rows_bytes / p.region_bytes):
//   [ s | o | eta replaced rows ] [ sc: eta_pad floats ] [ nid ] [ jorig ] [ mbarrier ]
// The relation row is NOT staged: each lane loads its chunks of p straight into registers (ld.global.nc, issued before
// the wait for the gather, so the latency hides behind it) and keeps them until the gradient rows of s, p, o are formed.
// One row less per positive is what lets a 12th warp fit beside cfg2's 11 (12 x (12 x 1600 + 160) B = 226.9 KB of the 227 KB a
// block may use).
// Gradient rows leave the SM as red.global.add.v4.f32 straight from registers.  Sending part of them down the copy
// engine's road instead (g*Q staged over the gathered row with st.shared.v4, one cp.reduce.async.bulk per row) was
// measured slower on cfg2 before the H100 port, for every second replaced row and for all of them.
// GATHER: the owner-computes path (kge_train_bucket.cu) -- instead of scattering g * Q into each replaced row, every
// corruption leaves (its entity, the kept-side entity, the relation and side, g) in its entity's bucket, at the slot the
// pre-pass ranked it to; the bucket sum forms the rows afterwards.  Everything else is the same kernel.
template <int HALVES, int NIT, int THREADS, bool GATHER>
__global__ void __launch_bounds__(THREADS) kge_train_res_kernel(const TrainParams p)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    KGE_KEEP32(warp);
    KGE_KEEP32(lane);
    uint32_t rows_s = smem_u32(smem_raw) + (uint32_t)warp * (uint32_t)p.region_bytes;
    uint32_t sc_s = rows_s + (uint32_t)p.rows_bytes;
    uint32_t nid_s = sc_s + 4u * (uint32_t)p.eta_pad;
    uint32_t jor_s = nid_s + 4u * (uint32_t)p.eta_pad;
    uint32_t bar_s = jor_s + 4u * (uint32_t)p.eta_pad;
    KGE_KEEP32(rows_s); KGE_KEEP32(sc_s); KGE_KEEP32(nid_s); KGE_KEEP32(jor_s); KGE_KEEP32(bar_s);
    float *const sc = reinterpret_cast<float *>(smem_raw + (size_t)warp * p.region_bytes + p.rows_bytes);  // for loss_and_dscores

    if (lane == 0) mbar_init_s(bar_s, 1);
    fence_mbar_init();
    fence_proxy_async_smem();
    __syncthreads();

    int ld = p.ld, eta = p.eta;
    const int nch = p.kp >> 2;
    uint32_t lwB = (uint32_t)p.slot_floats * 4u;  // bytes between rows of the slot
    uint32_t hsB = (uint32_t)p.kp * 4u;           // bytes between the real and the imaginary half of a row (slot and HBM alike)
    uint32_t row_bytes = (uint32_t)ld * 4u;
    KGE_KEEP32(ld); KGE_KEEP32(eta); KGE_KEEP32(lwB); KGE_KEEP32(hsB); KGE_KEEP32(row_bytes);
    uint32_t off[NIT];  // this lane's byte offset inside a half, per chunk
    int live_i[NIT];
#pragma unroll
    for (int it = 0; it < NIT; ++it) {
        const int c = lane + 32 * it;
        live_i[it] = c < nch ? 1 : 0;
        off[it] = 16u * (uint32_t)min(c, nch - 1);
        KGE_KEEP32(off[it]);
        KGE_KEEP32(live_i[it]);
    }
    bool live[NIT];
#pragma unroll
    for (int it = 0; it < NIT; ++it) live[it] = live_i[it] != 0;
    float scale = p.score_scale;  // HolE 2/k, else 1
    KGE_KEEPF(scale);
    unsigned lt = (1u << lane) - 1u;
    KGE_KEEP32(lt);
    float *grad_ent = p.grad_ent;
    KGE_KEEP64(grad_ent);
    const bool stamping = p.stamp_ent != nullptr && p.mode != KGE_STEP_FORWARD_ONLY;
    uint32_t phase = 0u;
    double loss_acc = 0.0;
    // Hot-entity privatisation.  On a skewed graph a few entities own a large share of all subject / object slots (Zipf(1)
    // over 14.5 k entities: the first holds 10 %, the first two 15 %), and every one of those positives adds 100 float4 to
    // the SAME gradient row: ~42,000 atomics per 128-byte line per step, which the L2 serialises per address -- measurably
    // slower than the same kernel on uniformly drawn triples (measured before the H100 port).  The caller names up to KGE_HOT entities (kge_set_hot_entities; the facade
    // takes the most frequent ones of the training set); each warp sums their subject / object gradient rows in registers
    // over all the positives it processes and issues ONE set of REDs per hot row when it retires.
    int hot0 = p.hot_ent[0], hot1 = KGE_HOT > 1 ? p.hot_ent[1] : -1;
    KGE_KEEP32(hot0); KGE_KEEP32(hot1);
    float4 H0r[NIT], H0i[NIT], H1r[NIT], H1i[NIT];  // (the second set folds away when KGE_HOT == 1)
#pragma unroll
    for (int it = 0; it < NIT; ++it) H0r[it] = H0i[it] = H1r[it] = H1i[it] = f4zero();

    const long long n_warps = (long long)gridDim.x * (blockDim.x >> 5);
    // (measured and rejected before the H100 port: two or three positives per draw -- no gain / slower; requesting the next positive's triple after
    // the score pass, so that the top of a positive waits for nothing -- no gain on cfg2, slower on cfg3)
    float next_draw = 0.f;  // lane 0: this warp's draw from the positive counter (kge_train_common.cuh: dynamic assignment)
    for (long long i = (long long)blockIdx.x * (blockDim.x >> 5) + warp; i < p.B;
         i = p.sched ? n_warps + (long long)(unsigned)__shfl_sync(0xffffffffu, next_draw, 0) : i + n_warps) {
        if (p.sched && lane == 0) next_draw = sched_draw(p.sched);  // consumed by the loop increment, a whole positive later
        // ---- the positive, and its corruptions sorted by side as they are drawn (A3) ----
        int tv = 0;
        if (lane < 3) tv = __ldg(p.triples + 3 * i + lane);
        const int s_id = __shfl_sync(0xffffffffu, tv, 0), p_id = __shfl_sync(0xffffffffu, tv, 1), o_id = __shfl_sync(0xffffffffu, tv, 2);
        int keep = -1, repl = 0, bk_at = 0;
        if (lane < eta) {
            const unsigned long long r = (unsigned long long)lane * (unsigned long long)p.B + (unsigned long long)i;
            corruption_of(p, r, keep, repl);
            if constexpr (GATHER) bk_at = p.bk.off[repl] + p.bk.pos[r];  // consumed after the loss: the loads are long done
        }
        // slots [0, n0) replaced the subject (keep_subj == 0), slots [n0, eta) the object; jorig[slot] = j
        const unsigned m0 = __ballot_sync(0xffffffffu, keep == 0), m1 = __ballot_sync(0xffffffffu, keep == 1);
        const int n0 = __popc(m0);
        int slot = 0;  // this lane's corruption's slot
        if (lane < eta) {
            const int t = keep ? n0 + __popc(m1 & lt) : __popc(m0 & lt);
            slot = t;
            sts_i(nid_s + 4u * (uint32_t)t, repl);
            sts_i(jor_s + 4u * (uint32_t)t, lane);
            if (stamping) p.stamp_ent[repl] = p.stamp;  // lazy optimizer: row touched
        }
        if (stamping) {
            if (lane == 0) p.stamp_ent[s_id] = p.stamp;
            if (lane == 1) p.stamp_ent[o_id] = p.stamp;
            if (lane == 2 && p.stamp_rel) p.stamp_rel[p_id] = p.stamp;
        }
        __syncwarp();

        // ---- gather (A2): one bulk copy per row, s | p | o | replaced rows in slot order ----
        const int nrow = 2 + eta;
        if (lane == 0) mbar_expect_tx_s(bar_s, (uint32_t)nrow * row_bytes);
        __syncwarp();
        for (int r = lane; r < nrow; r += 32) {
            const int id = r == 0 ? s_id : r == 1 ? o_id : lds_i(nid_s + 4u * (uint32_t)(r - 2));
            bulk_load_s(rows_s + (uint32_t)r * lwB, p.ent + (size_t)id * ld, row_bytes, bar_s);
        }
        // this lane's chunks of the relation row, straight to registers
        float4 pr[NIT], pi[NIT];
        {
            const char *prow = reinterpret_cast<const char *>(p.rel + (size_t)p_id * ld);
#pragma unroll
            for (int it = 0; it < NIT; ++it) {
                pr[it] = __ldg(reinterpret_cast<const float4 *>(prow + off[it]));
                if constexpr (HALVES == 2) pi[it] = __ldg(reinterpret_cast<const float4 *>(prow + off[it] + hsB));
                if (!live[it]) { pr[it] = f4zero(); pi[it] = f4zero(); }  // every query vector carries a factor of p
            }
        }
        char *const gs_row = reinterpret_cast<char *>(grad_ent + (size_t)s_id * ld);
        char *const gp_row = reinterpret_cast<char *>(p.grad_rel + (size_t)p_id * ld);
        char *const go_row = reinterpret_cast<char *>(grad_ent + (size_t)o_id * ld);
        mbar_wait_s(bar_s, phase);
        phase ^= 1u;

        // ---- per-positive query vectors and the positive's score (A4) ----
        // side 0 (subject replaced): f = <r, Q0>;  side 1 (object replaced): f = <r, Q1>   (re / im parts for HALVES = 2)
        float4 Q0r[NIT], Q0i[NIT], Q1r[NIT], Q1i[NIT];
        float4 W0r[NIT], W0i[NIT], W1r[NIT], W1i[NIT];  // sum_j g_j r_j per side
        float P;
        {
            float4 acc = f4zero();
#pragma unroll
            for (int it = 0; it < NIT; ++it) {
                const uint32_t a = rows_s + off[it];
                if constexpr (HALVES == 2) {
                    const float4 sr = lds4(a), si = lds4(a + hsB);
                    const float4 orr = lds4(a + lwB), oi = lds4(a + lwB + hsB);
                    Q0r[it] = query_subj<2, 0>(pr[it], pi[it], orr, oi); Q0i[it] = query_subj<2, 1>(pr[it], pi[it], orr, oi);
                    Q1r[it] = query_obj<2, 0>(sr, si, pr[it], pi[it]); Q1i[it] = query_obj<2, 1>(sr, si, pr[it], pi[it]);
                    acc = f4fma(sr, Q0r[it], acc);
                    acc = f4fma(si, Q0i[it], acc);
                    W0i[it] = W1i[it] = f4zero();
                } else {
                    const float4 vs = lds4(a), vo = lds4(a + lwB);
                    Q0r[it] = query_subj<1, 0>(pr[it], pi[it], vo, vo);
                    Q1r[it] = query_obj<1, 0>(vs, vs, pr[it], pi[it]);
                    acc = f4fma(vs, Q0r[it], acc);
                }
                W0r[it] = W1r[it] = f4zero();
            }
            P = warp_sum(f4hsum(acc));
        }

        // ---- pass A: the eta corruption scores, four (then two) rows of one side per trip ----
        auto score_side = [&](int lo, int hi, const float4(&qr)[NIT], const float4(&qi)[NIT]) {
            int t = lo;
            for (; hi - t >= 3; t += 4) {
                const uint32_t r0 = rows_s + (uint32_t)(2 + t) * lwB, r1 = r0 + lwB, r2 = r1 + lwB;
                const uint32_t r3 = (t + 3 < hi) ? r2 + lwB : r2;  // a trip of three: the fourth row aliases the third and is dropped
                float4 a = f4zero(), b = f4zero(), c = f4zero(), d = f4zero();
#pragma unroll
                for (int it = 0; it < NIT; ++it) {
                    const uint32_t o = off[it];
                    a = f4fma(lds4(r0 + o), qr[it], a);
                    b = f4fma(lds4(r1 + o), qr[it], b);
                    c = f4fma(lds4(r2 + o), qr[it], c);
                    d = f4fma(lds4(r3 + o), qr[it], d);
                    if constexpr (HALVES == 2) {
                        a = f4fma(lds4(r0 + o + hsB), qi[it], a);
                        b = f4fma(lds4(r1 + o + hsB), qi[it], b);
                        c = f4fma(lds4(r2 + o + hsB), qi[it], c);
                        d = f4fma(lds4(r3 + o + hsB), qi[it], d);
                    }
                }
                const float v = warp_sum4t(f4hsum(a), f4hsum(b), f4hsum(c), f4hsum(d), lane);  // lanes [8q, 8q+8) hold row q's sum
                const int q = lane >> 3;
                if ((lane & 7) == 0 && t + q < hi) sts_f(sc_s + 4u * (uint32_t)(t + q), v);
            }
            if (t < hi) {  // one or two rows left
                const bool has_b = t + 1 < hi;
                const uint32_t ra = rows_s + (uint32_t)(2 + t) * lwB, rb = has_b ? ra + lwB : ra;
                float4 a = f4zero(), b = f4zero();
#pragma unroll
                for (int it = 0; it < NIT; ++it) {
                    const uint32_t o = off[it];
                    a = f4fma(lds4(ra + o), qr[it], a);
                    b = f4fma(lds4(rb + o), qr[it], b);
                    if constexpr (HALVES == 2) {
                        a = f4fma(lds4(ra + o + hsB), qi[it], a);
                        b = f4fma(lds4(rb + o + hsB), qi[it], b);
                    }
                }
                float pa = f4hsum(a), pb = f4hsum(b);
                warp_sum2(pa, pb);
                if (lane == 0) {
                    sts_f(sc_s + 4u * (uint32_t)t, pa);
                    if (has_b) sts_f(sc_s + 4u * (uint32_t)(t + 1), pb);
                }
            }
        };
        score_side(0, n0, Q0r, Q0i);
        score_side(n0, eta, Q1r, Q1i);
        __syncwarp();

        // ---- loss and dL/dscore (A5) ----
        float dP;
        if (p.mode != KGE_STEP_BACKWARD_EXT) {
            if (scale != 1.f) {
                if (lane < eta) sc[lane] *= scale;
                __syncwarp();
            }
            if (p.scores_neg && lane < eta) p.scores_neg[(size_t)lds_i(jor_s + 4u * (uint32_t)lane) * p.B + i] = sc[lane];
            if (p.scores_pos && lane == 0) p.scores_pos[i] = scale * P;
            if (p.mode == KGE_STEP_FORWARD_ONLY) { __syncwarp(); continue; }
            const float li = loss_and_dscores(p, scale * P, sc, lane, &dP);
            if (lane == 0) loss_acc += (double)li;
        } else {
            if (lane < eta) sc[lane] = p.dneg[(size_t)lds_i(jor_s + 4u * (uint32_t)lane) * p.B + i];
            dP = p.dpos[i];
        }
        __syncwarp();
        if constexpr (GATHER) {
            if (lane < eta) {  // the g of red_row below, handed to the bucket sum
                p.bk.g[bk_at] = scale * lds_f(sc_s + 4u * (uint32_t)slot);
                p.bk.eid[bk_at] = repl;
                p.bk.other[bk_at] = keep ? s_id : o_id;
                p.bk.rel[bk_at] = p_id | (keep ? (int)0x80000000u : 0);
            }
        }

        // ---- pass B: gradient rows of the replaced entities, two rows of one side per trip; W += g * row ----
        // gradient REDs of one replaced row: g * Q at the lane's chunks.  One 64-bit base per half; chunk it sits 512*it bytes
        // further (off[it] = off[0] + 512*it wherever live[it]), which the RED takes as an immediate offset.
        auto red_row = [&](int id, float g, const float4(&qr)[NIT], const float4(&qi)[NIT]) {
            if (!live[0]) return;
            char *const g0 = reinterpret_cast<char *>(grad_ent + (size_t)id * ld) + off[0];
            char *const g1 = g0 + hsB;
#pragma unroll
            for (int it = 0; it < NIT; ++it) {
                if (!live[it]) break;
                red_repl_v4(reinterpret_cast<float *>(g0 + 512 * it), g * qr[it]);
                if constexpr (HALVES == 2) red_repl_v4(reinterpret_cast<float *>(g1 + 512 * it), g * qi[it]);
            }
        };
        auto grad_side = [&](int lo, int hi, const float4(&qr)[NIT], const float4(&qi)[NIT], float4(&Wr)[NIT], float4(&Wi)[NIT]) {
            for (int t = lo; t < hi; t += 2) {
                const bool has_b = t + 1 < hi;
                const uint32_t tb = (uint32_t)(has_b ? t + 1 : t);
                const uint32_t ra = rows_s + (uint32_t)(2 + t) * lwB, rb = rows_s + (2u + tb) * lwB;
                const float ga = scale * lds_f(sc_s + 4u * (uint32_t)t);
                const float gb = has_b ? scale * lds_f(sc_s + 4u * tb) : 0.f;
                const int ida = lds_i(nid_s + 4u * (uint32_t)t), idb = lds_i(nid_s + 4u * tb);
#pragma unroll
                for (int it = 0; it < NIT; ++it) {
                    const uint32_t o = off[it];
                    const float4 ar = lds4(ra + o), br = lds4(rb + o);
                    Wr[it] = f4fma(ga, ar, Wr[it]);
                    Wr[it] = f4fma(gb, br, Wr[it]);
                    if constexpr (HALVES == 2) {
                        const float4 ai = lds4(ra + o + hsB), bi = lds4(rb + o + hsB);
                        Wi[it] = f4fma(ga, ai, Wi[it]);
                        Wi[it] = f4fma(gb, bi, Wi[it]);
                    }
                }
                if constexpr (!GATHER) {
                    red_row(ida, ga, qr, qi);
                    if (has_b) red_row(idb, gb, qr, qi);
                }
            }
        };
        grad_side(0, n0, Q0r, Q0i, W0r, W0i);
        grad_side(n0, eta, Q1r, Q1i, W1r, W1i);

        // ---- gradient rows of s, p, o: bilinearity folds every corruption's share into W ----
        {
            const float gP = scale * dP;
#pragma unroll
            for (int it = 0; it < NIT; ++it) {
                if (!live[it]) continue;
                const uint32_t o = off[it], a = rows_s + o;
                if constexpr (HALVES == 2) {
                    const float4 sr = lds4(a), si = lds4(a + hsB);
                    const float4 orr = lds4(a + lwB), oi = lds4(a + lwB + hsB);
                    const float4 Ur = f4fma(gP, sr, W0r[it]), Ui = f4fma(gP, si, W0i[it]);    // everything that sat in the subject slot
                    const float4 Xr = f4fma(gP, orr, W1r[it]), Xi = f4fma(gP, oi, W1i[it]);   // everything that sat in the object slot
                    const float4 gsr = query_subj<2, 0>(pr[it], pi[it], Xr, Xi), gsi = query_subj<2, 1>(pr[it], pi[it], Xr, Xi);  // d/ds f(s,p,X)
                    const float4 gor = query_obj<2, 0>(Ur, Ui, pr[it], pi[it]), goi = query_obj<2, 1>(Ur, Ui, pr[it], pi[it]);    // d/do f(U,p,o)
                    if (s_id == hot0) { H0r[it] = H0r[it] + gsr; H0i[it] = H0i[it] + gsi; }
                    else if (KGE_HOT > 1 && s_id == hot1) { H1r[it] = H1r[it] + gsr; H1i[it] = H1i[it] + gsi; }
                    else { red4(gs_row, o, gsr); red4(gs_row, o + hsB, gsi); }
                    if (o_id == hot0) { H0r[it] = H0r[it] + gor; H0i[it] = H0i[it] + goi; }
                    else if (KGE_HOT > 1 && o_id == hot1) { H1r[it] = H1r[it] + gor; H1i[it] = H1i[it] + goi; }
                    else { red4(go_row, o, gor); red4(go_row, o + hsB, goi); }
                    red4(gp_row, o, trilinear_grad_p<2, 0>(sr, si, orr, oi, Ur, Ui, W1r[it], W1i[it]));
                    red4(gp_row, o + hsB, trilinear_grad_p<2, 1>(sr, si, orr, oi, Ur, Ui, W1r[it], W1i[it]));
                } else {
                    const float4 vs = lds4(a), vo = lds4(a + lwB);
                    const float4 U = f4fma(gP, vs, W0r[it]), X = f4fma(gP, vo, W1r[it]);
                    const float4 gsr = query_subj<1, 0>(pr[it], pi[it], X, X), gor = query_obj<1, 0>(U, U, pr[it], pi[it]);
                    if (s_id == hot0) H0r[it] = H0r[it] + gsr;
                    else if (KGE_HOT > 1 && s_id == hot1) H1r[it] = H1r[it] + gsr;
                    else red4(gs_row, o, gsr);
                    if (o_id == hot0) H0r[it] = H0r[it] + gor;
                    else if (KGE_HOT > 1 && o_id == hot1) H1r[it] = H1r[it] + gor;
                    else red4(go_row, o, gor);
                    red4(gp_row, o, trilinear_grad_p<1, 0>(vs, vs, vo, vo, U, U, W1r[it], W1r[it]));
                }
            }
        }
        __syncwarp();  // every lane has read the slot before the next positive's gather overwrites it
    }
    sched_retire(p.sched, n_warps, lane);
    // retire: this warp's share of the hot rows (zeros when it met none of them: skip)
    if (p.mode != KGE_STEP_FORWARD_ONLY) {
#pragma unroll
        for (int h = 0; h < KGE_HOT; ++h) {
            const int id = h ? hot1 : hot0;
            if (id < 0) continue;
            char *const row = reinterpret_cast<char *>(grad_ent + (size_t)id * ld);
#pragma unroll
            for (int it = 0; it < NIT; ++it) {
                if (!live[it]) continue;
                red4(row, off[it], h ? H1r[it] : H0r[it]);
                if constexpr (HALVES == 2) red4(row, off[it] + hsB, h ? H1i[it] : H0i[it]);
            }
        }
    }
    if (p.loss_out && p.mode == KGE_STEP_FUSED && lane == 0 && loss_acc != 0.0) atomicAdd(p.loss_out, loss_acc);
}

// ---- host side -------------------------------------------------------------------------------------------------------------
cudaError_t launch_train_res(const TrainParams &p, int nit, const TrainSlot &slot, int sm_count, cudaStream_t st)
{
    return dispatch_trilinear_shape(p.model, nit, [&](auto halves, auto nits) {
        constexpr int THREADS = KGE_TRAIN_THREADS(KGE_COMPLEX, nits);
        return launch_persistent(p.bk.g ? kge_train_res_kernel<halves, nits, THREADS, true> : kge_train_res_kernel<halves, nits, THREADS, false>,
                                 p, slot, sm_count, st);
    });
}

}  // namespace kge
