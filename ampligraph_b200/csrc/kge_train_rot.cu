// kge_train_rot.cu -- the RotatE fast path of the fused training step (sm_90a).
//
// Same contract as kge_train_kernel<KGE_ROTATE> (kge_train.cu; reference: train_step ScoringBasedEmbeddingModel.py:370-429 ->
// EmbeddingLookupLayer.call, CorruptionGenerationLayerTrain.call, RotatE._compute_scores RotatE.py:62-104, the five losses,
// tape.gradient), specialised the way kge_train_res.cu specialises the trilinear models, for the shape cfg4 has: one column
// window (k <= 256), a single (not row-sharded) table, any eta.  After the scorer had been put on an instruction budget the
// general kernel was (profiled before the H100 port) latency-bound at 2 warps per scheduler with a third of every inner loop spent on addressing
// (DESIGN.md 3.1); what this kernel does differently:
//   * s, o and the rotation row of the positive go STRAIGHT TO REGISTERS (ld.global.nc, coalesced 16 B per lane): everything
//     the two passes need of them is y = R(phi) s, o, cos, sin, which live in registers anyway.  The shared-memory slot then
//     holds only replaced rows, so the same 28 KB per warp take groups of 8 corruptions instead of 7 (cfg4: 4 groups
//     instead of 5), or the whole positive when 2G >= eta;
//   * the gradient pass starts on the TWO groups the score pass left in the buffers and re-gathers only the others, each
//     into the buffer that has just been consumed (the general kernel re-gathers all but the last);
//   * explicit 32-bit shared addresses, loop invariants kept in registers (KGE_KEEP*), one 64-bit gradient base per replaced
//     row with the second chunk and the imaginary half as immediate / register offsets of the RED.
// The per-element arithmetic is the general kernel's: both compute RotatE with the rot_* functions of
// kge_train_common.cuh, so both produce the same scores bit for bit; gradients differ only in the order of the fp32
// atomics (tests/test_gpu_parity.py::test_resident_fast_path_equals_general_kernel).
#include "kge_train_common.cuh"

namespace kge {

namespace {

// 16-byte read-only load that stays where it is written (asm volatile: the compiler may not sink it to its first use)
__device__ __forceinline__ float4 ldg4_nc(const char *p)
{
    float4 v;
    asm volatile("ld.global.nc.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
    return v;
}

}  // namespace

// Lane l owns float4 chunks c = l + 32*it (it < NIT) of every half-row; lanes past the end of the row read its last chunk,
// are masked arithmetically in the scores (nlive) and never store.
// Shared-memory slot of a warp (kge_create: the RotatE TrainSlot, p.rows_bytes / p.region_bytes):
//   [ nbuf group buffers of G rows ] [ sc: eta_pad floats ] [ nid ] [ jorig ] [ side: scratch ] [ 2 mbarriers ]
template <int NIT>
__global__ void __launch_bounds__(256) kge_train_rot_kernel(const TrainParams p)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    KGE_KEEP32(warp);
    KGE_KEEP32(lane);
    uint32_t rows_s = smem_u32(smem_raw) + (uint32_t)warp * (uint32_t)p.region_bytes;
    uint32_t sc_s = rows_s + (uint32_t)p.rows_bytes;
    uint32_t nid_s = sc_s + 4u * (uint32_t)p.eta_pad;
    uint32_t jor_s = nid_s + 4u * (uint32_t)p.eta_pad;
    uint32_t side_s = jor_s + 4u * (uint32_t)p.eta_pad;
    uint32_t bar_s = side_s + 4u * (uint32_t)p.eta_pad;  // two mbarriers, 8 bytes each
    KGE_KEEP32(rows_s); KGE_KEEP32(sc_s); KGE_KEEP32(nid_s); KGE_KEEP32(jor_s); KGE_KEEP32(side_s); KGE_KEEP32(bar_s);
    float *const sc = reinterpret_cast<float *>(smem_raw + (size_t)warp * p.region_bytes + p.rows_bytes);  // for loss_and_dscores

    if (lane == 0) { mbar_init_s(bar_s, 1); mbar_init_s(bar_s + 8u, 1); }
    fence_mbar_init();
    fence_proxy_async_smem();
    __syncthreads();

    int ld = p.ld, eta = p.eta, G = p.G;
    const int nch = p.kp >> 2;
    const int n_groups = (eta + G - 1) / G;
    uint32_t lwB = (uint32_t)p.slot_floats * 4u;  // bytes between rows of the slot
    uint32_t hsB = (uint32_t)p.kp * 4u;           // bytes between the real and the imaginary half of a row (slot and HBM alike)
    uint32_t row_bytes = (uint32_t)ld * 4u;
    KGE_KEEP32(ld); KGE_KEEP32(eta); KGE_KEEP32(G); KGE_KEEP32(lwB); KGE_KEEP32(hsB); KGE_KEEP32(row_bytes);
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
    float nlive[NIT];  // -1 / 0: the arithmetic lane mask of the score sums
#pragma unroll
    for (int it = 0; it < NIT; ++it) { live[it] = live_i[it] != 0; nlive[it] = live[it] ? -1.f : 0.f; }
    unsigned lt = (1u << lane) - 1u;
    KGE_KEEP32(lt);
    float *grad_ent = p.grad_ent;
    KGE_KEEP64(grad_ent);
    const bool stamping = p.stamp_ent != nullptr && p.mode != KGE_STEP_FORWARD_ONLY;
    const float inv_div = p.inv_div;
    uint32_t phase0 = 0u, phase1 = 0u;
    double loss_acc = 0.0;

    // gather of group g (slots [g*G, g*G + gsz)) into buffer b: one bulk copy per row, completion on the buffer's mbarrier
    auto issue = [&](int g, int b) {
        const int j0 = g * G, gsz = min(G, eta - j0);
        if (lane == 0) mbar_expect_tx_s(bar_s + 8u * (uint32_t)b, (uint32_t)gsz * row_bytes);
        __syncwarp();
        for (int r = lane; r < gsz; r += 32)
            bulk_load_s(rows_s + (uint32_t)(b * G + r) * lwB, p.ent + (size_t)lds_i(nid_s + 4u * (uint32_t)(j0 + r)) * ld, row_bytes,
                        bar_s + 8u * (uint32_t)b);
    };
    auto wait = [&](int b) {
        if (b) { mbar_wait_s(bar_s + 8u, phase1); phase1 ^= 1u; }
        else { mbar_wait_s(bar_s, phase0); phase0 ^= 1u; }
    };

    const long long n_warps = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long i = (long long)blockIdx.x * (blockDim.x >> 5) + warp; i < p.B; i += n_warps) {
        // ---- the positive, and its corruptions sorted by side as they are drawn (A3) ----
        int tv = 0;
        if (lane < 3) tv = __ldg(p.triples + 3 * i + lane);
        const int s_id = __shfl_sync(0xffffffffu, tv, 0), p_id = __shfl_sync(0xffffffffu, tv, 1), o_id = __shfl_sync(0xffffffffu, tv, 2);
        // this lane's chunks of s, the rotation row [cos | sin] and o, straight to registers -- requested FIRST, so that their
        // latency hides behind the corruption draws below (long-scoreboard was the top stall with the loads placed
        // where they are consumed, profiled before the H100 port)
        float4 sr[NIT], si[NIT], C[NIT], Sn[NIT], Or_[NIT], Oi[NIT];
        {
            const char *srow = reinterpret_cast<const char *>(p.ent + (size_t)s_id * ld);
            const char *prow = reinterpret_cast<const char *>(p.rel + (size_t)p_id * ld);
            const char *orow = reinterpret_cast<const char *>(p.ent + (size_t)o_id * ld);
#pragma unroll
            for (int it = 0; it < NIT; ++it) {
                sr[it] = ldg4_nc(srow + off[it]); si[it] = ldg4_nc(srow + off[it] + hsB);
                C[it] = ldg4_nc(prow + off[it]); Sn[it] = ldg4_nc(prow + off[it] + hsB);
                Or_[it] = ldg4_nc(orow + off[it]); Oi[it] = ldg4_nc(orow + off[it] + hsB);
            }
        }
        int n0 = 0;
        for (int base = 0; base < eta; base += 32) {
            const int j = base + lane;
            int keep = -1, repl = 0;
            if (j < eta) {
                corruption_of(p, (unsigned long long)j * (unsigned long long)p.B + (unsigned long long)i, keep, repl);
                sts_i(side_s + 4u * (uint32_t)j, keep);  // keep_subj = 1 -> object replaced -> side 1
                sts_i(sc_s + 4u * (uint32_t)j, repl);
                if (stamping) p.stamp_ent[repl] = p.stamp;  // lazy optimizer: row touched
            }
            n0 += __popc(__ballot_sync(0xffffffffu, keep == 0));
        }
        __syncwarp();
        {   // slots [0, n0) replaced the subject, slots [n0, eta) the object; jorig[slot] = j
            int c0 = 0, c1 = n0;
            for (int base = 0; base < eta; base += 32) {
                const int j = base + lane;
                const int keep = (j < eta) ? lds_i(side_s + 4u * (uint32_t)j) : -1;
                const unsigned m0 = __ballot_sync(0xffffffffu, keep == 0), m1 = __ballot_sync(0xffffffffu, keep == 1);
                if (j < eta) {
                    const int t = keep ? c1 + __popc(m1 & lt) : c0 + __popc(m0 & lt);
                    sts_i(nid_s + 4u * (uint32_t)t, lds_i(sc_s + 4u * (uint32_t)j));
                    sts_i(jor_s + 4u * (uint32_t)t, j);
                }
                c0 += __popc(m0);
                c1 += __popc(m1);
            }
        }
        if (stamping) {
            if (lane == 0) p.stamp_ent[s_id] = p.stamp;
            if (lane == 1) p.stamp_ent[o_id] = p.stamp;
            if (lane == 2 && p.stamp_rel) p.stamp_rel[p_id] = p.stamp;
        }
        __syncwarp();

        // ---- gather (A2): the first group by the copy engine; per-positive state from the rows requested above ----
        issue(0, 0);
        float4 Yr[NIT], Yi[NIT];
        float4 Zor[NIT], Zoi[NIT], Zsr[NIT], Zsi[NIT], Aphi[NIT];
        float P;
        {
            float acc = 0.f;
#pragma unroll
            for (int it = 0; it < NIT; ++it) {
                if (!live[it]) { sr[it] = si[it] = f4zero(); C[it] = Sn[it] = Or_[it] = Oi[it] = f4zero(); }
                Yr[it] = rot_rotate<0>(sr[it], si[it], C[it], Sn[it]);
                Yi[it] = rot_rotate<1>(sr[it], si[it], C[it], Sn[it]);
                Zor[it] = Zoi[it] = Zsr[it] = Zsi[it] = Aphi[it] = f4zero();
                acc = fmaf(rot_modsum(Yr[it] - Or_[it], Yi[it] - Oi[it]), nlive[it], acc);
            }
            P = warp_sum(acc);
        }
        char *const gs_row = reinterpret_cast<char *>(grad_ent + (size_t)s_id * ld);
        char *const gp_row = reinterpret_cast<char *>(p.grad_rel + (size_t)p_id * ld);
        char *const go_row = reinterpret_cast<char *>(grad_ent + (size_t)o_id * ld);

        // ---- pass A: scores, group by group, next group prefetched into the other buffer (A4) ----
        for (int g = 0; g < n_groups; ++g) {
            const int buf = g & 1, j0 = g * G, gsz = min(G, eta - j0);
            if (g + 1 < n_groups) issue(g + 1, buf ^ 1);  // every lane finished group g-1 (the __syncwarp below)
            wait(buf);
            const uint32_t grp = rows_s + (uint32_t)(buf * G) * lwB;
            const int e0 = min(n0, j0 + gsz), b1 = max(n0, j0);  // [j0, e0) replaced the subject, [b1, j0+gsz) the object
            for (int t = j0; t < e0; t += 2) {  // residual = R(phi) r - o
                const bool has_b = t + 1 < e0;
                const uint32_t ra = grp + (uint32_t)(t - j0) * lwB, rb = has_b ? ra + lwB : ra;
                float a = 0.f, b = 0.f;
#pragma unroll
                for (int it = 0; it < NIT; ++it) {
                    const float4 ar = lds4(ra + off[it]), ai = lds4(ra + off[it] + hsB);
                    const float4 br = lds4(rb + off[it]), bi = lds4(rb + off[it] + hsB);
                    const float4 e0r = rot_residual_subj<0>(ar, ai, C[it], Sn[it], Or_[it], Oi[it]);
                    const float4 e0i = rot_residual_subj<1>(ar, ai, C[it], Sn[it], Or_[it], Oi[it]);
                    const float4 e1r = rot_residual_subj<0>(br, bi, C[it], Sn[it], Or_[it], Oi[it]);
                    const float4 e1i = rot_residual_subj<1>(br, bi, C[it], Sn[it], Or_[it], Oi[it]);
                    a = fmaf(rot_modsum(e0r, e0i), nlive[it], a);
                    b = fmaf(rot_modsum(e1r, e1i), nlive[it], b);
                }
                const float v = warp_sum2t(a, b, lane);
                if ((lane & 15) == 0 && (lane == 0 || has_b)) sts_f(sc_s + 4u * (uint32_t)(t + (lane ? 1 : 0)), v);
            }
            for (int t = b1; t < j0 + gsz; t += 2) {  // residual = y - r
                const bool has_b = t + 1 < j0 + gsz;
                const uint32_t ra = grp + (uint32_t)(t - j0) * lwB, rb = has_b ? ra + lwB : ra;
                float a = 0.f, b = 0.f;
#pragma unroll
                for (int it = 0; it < NIT; ++it) {
                    const float4 ar = lds4(ra + off[it]), ai = lds4(ra + off[it] + hsB);
                    const float4 br = lds4(rb + off[it]), bi = lds4(rb + off[it] + hsB);
                    a = fmaf(rot_modsum(Yr[it] - ar, Yi[it] - ai), nlive[it], a);
                    b = fmaf(rot_modsum(Yr[it] - br, Yi[it] - bi), nlive[it], b);
                }
                const float v = warp_sum2t(a, b, lane);
                if ((lane & 15) == 0 && (lane == 0 || has_b)) sts_f(sc_s + 4u * (uint32_t)(t + (lane ? 1 : 0)), v);
            }
            __syncwarp();
        }

        // ---- loss and dL/dscore (A5) ----
        float dP;
        if (p.mode != KGE_STEP_BACKWARD_EXT) {
            if (p.scores_neg)
                for (int t = lane; t < eta; t += 32) p.scores_neg[(size_t)lds_i(jor_s + 4u * (uint32_t)t) * p.B + i] = sc[t];
            if (p.scores_pos && lane == 0) p.scores_pos[i] = P;
            if (p.mode == KGE_STEP_FORWARD_ONLY) { __syncwarp(); continue; }
            const float li = loss_and_dscores(p, P, sc, lane, &dP);
            if (lane == 0) loss_acc += (double)li;
        } else {
            for (int t = lane; t < eta; t += 32) sc[t] = p.dneg[(size_t)lds_i(jor_s + 4u * (uint32_t)t) * p.B + i];
            dP = p.dpos[i];
        }
        __syncwarp();

        // ---- pass B: gradients, last group first.  The buffers still hold the last two groups; group g-2 is re-gathered into
        // group g's buffer as soon as group g has been consumed ----
        for (int g = n_groups - 1; g >= 0; --g) {
            const int buf = g & 1, j0 = g * G, gsz = min(G, eta - j0);
            if (g < n_groups - 2) wait(buf);
            const uint32_t grp = rows_s + (uint32_t)(buf * G) * lwB;
            const int e0 = min(n0, j0 + gsz), b1 = max(n0, j0);
            // two rows of one side per trip (four independent chains with NIT = 2); a lone last row is paired with itself
            // at weight 0 and not stored
            for (int t = j0; t < e0; t += 2) {  // subject replaced: residual = R(phi) r - o ; df/dr = -R(-phi)(a,b)
                const bool has_b = t + 1 < e0;
                const uint32_t tb = (uint32_t)(has_b ? t + 1 : t);
                const uint32_t ra = grp + (uint32_t)(t - j0) * lwB, rb = has_b ? ra + lwB : ra;
                const float ga = lds_f(sc_s + 4u * (uint32_t)t), gb = has_b ? lds_f(sc_s + 4u * tb) : 0.f;
                char *const ga0 = reinterpret_cast<char *>(grad_ent + (size_t)lds_i(nid_s + 4u * (uint32_t)t) * ld) + off[0];
                char *const gb0 = reinterpret_cast<char *>(grad_ent + (size_t)lds_i(nid_s + 4u * tb) * ld) + off[0];
#pragma unroll
                for (int it = 0; it < NIT; ++it) {
                    const float4 ar = lds4(ra + off[it]), ai = lds4(ra + off[it] + hsB);
                    const float4 br = lds4(rb + off[it]), bi = lds4(rb + off[it] + hsB);
                    const float4 yar = rot_rotate<0>(ar, ai, C[it], Sn[it]), yai = rot_rotate<1>(ar, ai, C[it], Sn[it]);  // R(phi) r
                    const float4 ybr = rot_rotate<0>(br, bi, C[it], Sn[it]), ybi = rot_rotate<1>(br, bi, C[it], Sn[it]);
                    float4 a, b, c, d;
                    rot_unit(yar - Or_[it], yai - Oi[it], ga, a, b);
                    rot_unit(ybr - Or_[it], ybi - Oi[it], gb, c, d);
                    Zsr[it] = Zsr[it] + a; Zsi[it] = Zsi[it] + b;
                    Zsr[it] = Zsr[it] + c; Zsi[it] = Zsi[it] + d;
                    Aphi[it] = rot_dphi(a, b, yar, yai, Aphi[it]);
                    Aphi[it] = rot_dphi(c, d, ybr, ybi, Aphi[it]);
                    if (live[it]) {
                        red_add_v4(reinterpret_cast<float *>(ga0 + 512 * it), rot_back<0>(a, b, C[it], Sn[it]));
                        red_add_v4(reinterpret_cast<float *>(ga0 + hsB + 512 * it), rot_back<1>(a, b, C[it], Sn[it]));
                    }
                    if (live[it] && has_b) {
                        red_add_v4(reinterpret_cast<float *>(gb0 + 512 * it), rot_back<0>(c, d, C[it], Sn[it]));
                        red_add_v4(reinterpret_cast<float *>(gb0 + hsB + 512 * it), rot_back<1>(c, d, C[it], Sn[it]));
                    }
                }
            }
            for (int t = b1; t < j0 + gsz; t += 2) {  // object replaced: residual = y(s) - r ; df/dr = +(a,b)
                const bool has_b = t + 1 < j0 + gsz;
                const uint32_t tb = (uint32_t)(has_b ? t + 1 : t);
                const uint32_t ra = grp + (uint32_t)(t - j0) * lwB, rb = has_b ? ra + lwB : ra;
                const float ga = lds_f(sc_s + 4u * (uint32_t)t), gb = has_b ? lds_f(sc_s + 4u * tb) : 0.f;
                char *const ga0 = reinterpret_cast<char *>(grad_ent + (size_t)lds_i(nid_s + 4u * (uint32_t)t) * ld) + off[0];
                char *const gb0 = reinterpret_cast<char *>(grad_ent + (size_t)lds_i(nid_s + 4u * tb) * ld) + off[0];
#pragma unroll
                for (int it = 0; it < NIT; ++it) {
                    const float4 ar = lds4(ra + off[it]), ai = lds4(ra + off[it] + hsB);
                    const float4 br = lds4(rb + off[it]), bi = lds4(rb + off[it] + hsB);
                    float4 a, b, c, d;
                    rot_unit(Yr[it] - ar, Yi[it] - ai, ga, a, b);
                    rot_unit(Yr[it] - br, Yi[it] - bi, gb, c, d);
                    Zor[it] = Zor[it] + a; Zoi[it] = Zoi[it] + b;
                    Zor[it] = Zor[it] + c; Zoi[it] = Zoi[it] + d;
                    if (live[it]) {
                        red_add_v4(reinterpret_cast<float *>(ga0 + 512 * it), a);
                        red_add_v4(reinterpret_cast<float *>(ga0 + hsB + 512 * it), b);
                    }
                    if (live[it] && has_b) {
                        red_add_v4(reinterpret_cast<float *>(gb0 + 512 * it), c);
                        red_add_v4(reinterpret_cast<float *>(gb0 + hsB + 512 * it), d);
                    }
                }
            }
            __syncwarp();  // every lane has read group g: its buffer may be overwritten
            if (g >= 2) issue(g - 2, buf);
        }

        // ---- gradient rows of s, p, o ----
#pragma unroll
        for (int it = 0; it < NIT; ++it) {
            if (!live[it]) continue;
            float4 a, b;
            rot_unit(Yr[it] - Or_[it], Yi[it] - Oi[it], dP, a, b);
            const float4 Zr = a + Zor[it], Zi = b + Zoi[it];  // everything with y = R(phi) s
            red4(gs_row, off[it], rot_back<0>(Zr, Zi, C[it], Sn[it]));
            red4(gs_row, off[it] + hsB, rot_back<1>(Zr, Zi, C[it], Sn[it]));
            red4(go_row, off[it], a + Zsr[it]);
            red4(go_row, off[it] + hsB, b + Zsi[it]);
            // d/dtheta = (1/div) d/dphi in the first half of the relation row (the second half is allocated but unused, RotatE.py:76)
            red4(gp_row, off[it], inv_div * rot_dphi(Zr, Zi, Yr[it], Yi[it], Aphi[it]));
        }
        __syncwarp();  // the bookkeeping arrays are rewritten by the next positive
    }
    if (p.loss_out && p.mode == KGE_STEP_FUSED && lane == 0 && loss_acc != 0.0) atomicAdd(p.loss_out, loss_acc);
}

// ---- host side -------------------------------------------------------------------------------------------------------------
cudaError_t launch_train_rot(const TrainParams &p, int nit, const TrainSlot &slot, int sm_count, cudaStream_t st)
{
    if (nit <= 1) return launch_persistent(kge_train_rot_kernel<1>, p, slot, sm_count, st);
    if (nit == 2) return launch_persistent(kge_train_rot_kernel<2>, p, slot, sm_count, st);
    return cudaErrorInvalidValue;  // rows of 512+ floats per half stay on the general kernel (kge_create)
}

}  // namespace kge
