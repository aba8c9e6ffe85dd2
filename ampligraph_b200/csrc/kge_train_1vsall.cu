// kge_train_1vsall.cu -- 1vsAll training of the trilinear models (DistMult / ComplEx / HolE): the multiclass NLL of
// every positive against EVERY entity on one side (kge_one_vs_all_step; DESIGN.md 3.12).
//
// For a positive (s, p, o) and side o the logits are l_e = f(s, p, e) = scale * <x_e, q> over all entities e, with
// q = Q1(s, p) the query vector of kge_rank_qvec_kernel (side s: l_e = f(e, p, o), q = Q0(p, o)); scale is HolE's, 1
// otherwise.  Every logit is clipped to [-75, 75] (loss_functions.py:32-35) and the gradient is zero outside that range.
// With t the positive's own entity, w = 1 (reduction sum) or 1 / (n_ent - 1) (mean) and m the row's largest clipped
// logit:  D = w * sum_{e != t} exp(l_e - m) + exp(l_t - m),  loss = m + log(D) - l_t,
//         dL/dl_e = in_e * (w_e * exp(l_e - m) / D - [e == t]),  w_t = 1, w_e = w otherwise.
// Sum: logsumexp - l_t; mean: the reference's NLLMulticlass with the exp of the n_ent - 1 negatives averaged.
//
// Five passes per side, each a [B, ld] x [ld, n_ent]-shaped fp32 contraction on CUDA cores (FMA chains, no tensor
// cores); every CTA works on tiles of 32 queries x 32 entities, staged column chunk by column chunk with cp.async:
//   stats  (query tile x entity split): online max-subtracted (max, sum exp) of each row over its split, and l_t;
//   merge  (one thread per row): combines the splits, the row loss -> *loss, m and 1 / D per row;
//   dQ     (query tile x entity split): recomputes the logits, forms g, accumulates Gq = sum_e g_e x_e in shared memory
//          and writes its split's partial rows once;
//   dX     (entity tile, every query tile): recomputes the logits, accumulates sum_b g_be q_b in shared memory and adds
//          it to each of its grad_ent rows once (one owner per row: no atomics, deterministic);
//   chain  (one thread per row chunk): sums the split partials in order (scale included), and by linearity of f in the
//          query row forms the gradient rows of the positive's kept rows -- side o: d/ds = Q0(p, Gq), d/dp of f(s, p, Gq);
//          side s: d/do = Q1(Gq, p), d/dp of f(Gq, p, o) -- with the training kernels' own arithmetic
//          (kge_train_common.cuh), added with red.global.add like theirs.
// With embedding dropout (kge_dropout.cu; DESIGN.md 3.19) the passes read the side's dropped candidate table and the
// queries of its dropped query rows; dX adds into a zeroed workspace table that is masked into grad_cand afterwards, and
// kge_dropout.cu's chain pass replaces the one here.
// Every pass scores a (query, entity) pair with the same chain: one fma per column in ascending order, so the logits
// of the three passes that form them are bit-identical.
//
// KvsAll (kge_k_vs_all_step; DESIGN.md 3.13) trains each distinct (s, p) (side o) or (p, o) (side s) query against
// every entity with the multi-label NLL: target y'_e = (1 - eps) [e is a label] + eps / n_ent, weight w = 1 (sum) or
// 1 / n_ent (mean), loss = w * sum_e softplus(l_e) - y'_e l_e, dL/dl_e = in_e * w * (sigmoid(l_e) - y'_e).  The loss is
// element-wise, so a side is the dQ pass (which also adds the loss), the dX pass and the chain pass above, with the
// multi-label rule in place of the multiclass one.  The labels are a CSR (ascending ids per query); each 32 x 32 tile
// reads them as one 32-bit mask per query row, built in shared memory from the row's slice.
//
// Relation prediction as an auxiliary 1vsAll term (kge_one_vs_all_relation_step; DESIGN.md 3.14) is a third side,
// KGE_SIDE_P, whose candidates are the n_rel relation rows: l_r = f(s, r, o) = scale * <x_r, Qp(s, o)> with Qp = df/dp,
// the positive's relation the target, the row loss and dL/dl times the side's weight lambda.  It runs the same five
// passes; its dX pass is split over the query tiles too (n_rel / 32 relation tiles alone would leave most SMs idle), the
// partial rows summed in split order, and its chain pass adds d/ds = Q0(Gq, o) and d/do = Q1(s, Gq).
#include <math.h>

#include "kge_train_common.cuh"

namespace kge {

constexpr int OVA_T = 32;                       // queries per query tile = entities per entity tile
constexpr int OVA_DK = 32;                      // columns per staged chunk
constexpr int OVA_LDS = OVA_DK + 4;             // padded shared row: the per-thread 128-bit reads are conflict free
constexpr int OVA_THREADS = 256;
constexpr int OVA_CHUNK = OVA_T * OVA_LDS;      // floats of one staged chunk of 32 rows
constexpr int OVA_STAGE = 4 * OVA_CHUNK;        // two buffers of (query chunk, entity chunk)
constexpr int OVA_GS = OVA_T * (OVA_T + 1);     // the g tile [query][entity], padded rows
constexpr int OVA_TARGET_CTAS = 264;            // two CTAs on each of the H100's 132 SMs
constexpr int OVA_MAX_SPLITS = 64;

int one_vs_all_splits(long long B, long long n_ent)
{
    const long long n_qt = (B + OVA_T - 1) / OVA_T, n_et = (n_ent + OVA_T - 1) / OVA_T;
    long long s = n_qt > 0 ? (OVA_TARGET_CTAS + n_qt - 1) / n_qt : 1;
    if (s > OVA_MAX_SPLITS) s = OVA_MAX_SPLITS;
    if (s > n_et) s = n_et;
    return s < 1 ? 1 : (int)s;
}

size_t one_vs_all_smem_bytes(int ld) { return (OVA_STAGE + OVA_GS + (size_t)OVA_T * ld) * sizeof(float); }

// rows [r0, r0 + 32) x columns [c0, c0 + 32) of the [nrows, ld] matrix M -> dst (row stride OVA_LDS), zero past its ends
__device__ __forceinline__ void ova_stage(float *dst, const float *M, long long r0, long long nrows, int ld, int c0, int tid)
{
    const int r = tid >> 3, c = (tid & 7) * 4;
    const bool ok = r0 + r < nrows && c0 + c < ld;
    cp_async16(dst + r * OVA_LDS + c, ok ? M + (size_t)(r0 + r) * ld + c0 + c : M, ok);
}

__device__ __forceinline__ float4 ova_lds4(const float *p) { return *reinterpret_cast<const float4 *>(p); }
__device__ __forceinline__ float ova_dot4(float4 a, float4 b, float acc)
{
    acc = __fmaf_rn(a.x, b.x, acc);
    acc = __fmaf_rn(a.y, b.y, acc);
    acc = __fmaf_rn(a.z, b.z, acc);
    return __fmaf_rn(a.w, b.w, acc);
}

// acc[i][j] = <Q[q0 + 2 ty + i], X[e0 + tx + 16 j]> (ty = tid / 16, tx = tid % 16), zero for rows past nq / ne.
// Ends with a barrier: the caller may reuse `stage` and read what other threads wrote before the call.
__device__ __forceinline__ void ova_logits(const float *Q, long long q0, long long nq, const float *X, long long e0,
                                           long long ne, int ld, float *stage, int tid, float acc[2][2])
{
    const int ty = tid >> 4, tx = tid & 15;
    acc[0][0] = acc[0][1] = acc[1][0] = acc[1][1] = 0.f;
    const int nchunk = (ld + OVA_DK - 1) / OVA_DK;
    ova_stage(stage, Q, q0, nq, ld, 0, tid);
    ova_stage(stage + OVA_CHUNK, X, e0, ne, ld, 0, tid);
    cp_async_commit();
    for (int c = 0; c < nchunk; ++c) {
        const float *buf = stage + (c & 1) * 2 * OVA_CHUNK;
        if (c + 1 < nchunk) {
            float *nb = stage + ((c + 1) & 1) * 2 * OVA_CHUNK;
            ova_stage(nb, Q, q0, nq, ld, (c + 1) * OVA_DK, tid);
            ova_stage(nb + OVA_CHUNK, X, e0, ne, ld, (c + 1) * OVA_DK, tid);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        const float *qs = buf + 2 * ty * OVA_LDS, *xs = buf + OVA_CHUNK + tx * OVA_LDS;
#pragma unroll
        for (int k = 0; k < OVA_DK; k += 4) {
            const float4 a0 = ova_lds4(qs + k), a1 = ova_lds4(qs + OVA_LDS + k);
            const float4 b0 = ova_lds4(xs + k), b1 = ova_lds4(xs + 16 * OVA_LDS + k);
            acc[0][0] = ova_dot4(a0, b0, acc[0][0]);
            acc[0][1] = ova_dot4(a0, b1, acc[0][1]);
            acc[1][0] = ova_dot4(a1, b0, acc[1][0]);
            acc[1][1] = ova_dot4(a1, b1, acc[1][1]);
        }
        __syncthreads();
    }
}

// acc_s[o][:] += sum_r G(o, r) M[r0 + r][:] over the 32 rows of M from r0 (G(o, r) = gs[o][r], or gs[r][o] when
// TRANS); acc_s is [32, ld].  Thread (o = tid / 8, 4 columns) owns its part of acc_s.  Ends with a barrier.
template <bool TRANS>
__device__ __forceinline__ void ova_accumulate(float *acc_s, const float *gs, const float *M, long long r0, long long nrows,
                                               int ld, float *stage, int tid)
{
    const int o = tid >> 3, c4 = (tid & 7) * 4;
    const int nchunk = (ld + OVA_DK - 1) / OVA_DK;
    ova_stage(stage, M, r0, nrows, ld, 0, tid);
    cp_async_commit();
    for (int c = 0; c < nchunk; ++c) {
        const float *buf = stage + (c & 1) * OVA_CHUNK;
        if (c + 1 < nchunk) {
            ova_stage(stage + ((c + 1) & 1) * OVA_CHUNK, M, r0, nrows, ld, (c + 1) * OVA_DK, tid);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        const int col = c * OVA_DK + c4;
        if (col < ld) {
            float4 a = ova_lds4(acc_s + (size_t)o * ld + col);
#pragma unroll 8
            for (int r = 0; r < OVA_T; ++r) {
                const float g = TRANS ? gs[r * (OVA_T + 1) + o] : gs[o * (OVA_T + 1) + r];
                const float4 x = ova_lds4(buf + r * OVA_LDS + c4);
                a.x = __fmaf_rn(g, x.x, a.x);
                a.y = __fmaf_rn(g, x.y, a.y);
                a.z = __fmaf_rn(g, x.z, a.z);
                a.w = __fmaf_rn(g, x.w, a.w);
            }
            *reinterpret_cast<float4 *>(acc_s + (size_t)o * ld + col) = a;
        }
        __syncthreads();
    }
}

__device__ __forceinline__ float ova_clip(float acc, float scale, bool &in)
{
    const float l = scale * acc;
    in = l >= KGE_CLIP_LO && l <= KGE_CLIP_HI;
    return fminf(fmaxf(l, KGE_CLIP_LO), KGE_CLIP_HI);
}

// dL/dl of candidate e in a row with target t, max m, 1 / D = inv (times the side's weight: 1, or lambda for side p)
__device__ __forceinline__ float ova_grad(float acc, const OneVsAllSide &s, long long e, long long t, float m, float inv)
{
    bool in;
    const float l = ova_clip(acc, s.scale, in);
    if (!in) return 0.f;
    const float p = expf(l - m) * inv;
    return s.weight * (e == t ? p - 1.f : s.w * p);
}

__device__ __forceinline__ void ova_zero(float *a, int n, int tid)
{
    for (int i = tid * 4; i < n; i += OVA_THREADS * 4) *reinterpret_cast<float4 *>(a + i) = make_float4(0.f, 0.f, 0.f, 0.f);
}

// the entity-tile range [et0, et1) of split `split`
__device__ __forceinline__ void ova_split_range(const OneVsAllSide &s, int split, long long &et0, long long &et1)
{
    const long long n_et = (s.n_cand + OVA_T - 1) / OVA_T;
    et0 = split * n_et / s.nsplit;
    et1 = (split + 1) * n_et / s.nsplit;
}

__global__ void __launch_bounds__(OVA_THREADS) kge_ova_stats_kernel(const OneVsAllSide s)
{
    extern __shared__ __align__(16) float ova_sm[];
    const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15, split = blockIdx.y;
    const long long q0 = (long long)blockIdx.x * OVA_T;
    long long et0, et1;
    ova_split_range(s, split, et0, et1);
    long long tgt[2];
    float m[2], z[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const long long b = q0 + 2 * ty + i;
        tgt[i] = b < s.B ? s.triples[3 * b + s.col] : -1;
        m[i] = -INFINITY;
        z[i] = 0.f;
    }
    for (long long et = et0; et < et1; ++et) {
        const long long e0 = et * OVA_T;
        float acc[2][2];
        ova_logits(s.q, q0, s.B, s.cand, e0, s.n_cand, s.ld, ova_sm, tid, acc);
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const long long e = e0 + tx + 16 * j;
                if (tgt[i] < 0 || e >= s.n_cand) continue;
                bool in;
                const float l = ova_clip(acc[i][j], s.scale, in);
                if (e == tgt[i]) {  // the positive's own logit: counted in m, kept out of the sum
                    const long long b = q0 + 2 * ty + i;
                    s.lt[b] = l;
                    const float mn = fmaxf(m[i], l);
                    z[i] *= expf(m[i] - mn);
                    m[i] = mn;
                } else if (l > m[i]) {
                    z[i] = __fmaf_rn(z[i], expf(m[i] - l), 1.f);
                    m[i] = l;
                } else {
                    z[i] += expf(l - m[i]);
                }
            }
    }
    // the 16 threads of a query row are lanes of one half-warp
#pragma unroll
    for (int i = 0; i < 2; ++i) {
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) {
            const float m2 = __shfl_xor_sync(0xffffffffu, m[i], o), z2 = __shfl_xor_sync(0xffffffffu, z[i], o);
            const float mn = fmaxf(m[i], m2);
            z[i] = mn == -INFINITY ? 0.f : z[i] * expf(m[i] - mn) + z2 * expf(m2 - mn);
            m[i] = mn;
        }
        const long long b = q0 + 2 * ty + i;
        if (tx == 0 && b < s.B) {
            s.pm[split * s.B + b] = m[i];
            s.pz[split * s.B + b] = z[i];
        }
    }
}

__global__ void __launch_bounds__(256) kge_ova_merge_kernel(const OneVsAllSide s)
{
    const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    float loss = 0.f;
    if (b < s.B) {
        float m = -INFINITY, z = 0.f;
        for (int k = 0; k < s.nsplit; ++k) m = fmaxf(m, s.pm[k * s.B + b]);
        for (int k = 0; k < s.nsplit; ++k) {
            const float mk = s.pm[k * s.B + b];
            if (mk != -INFINITY) z += s.pz[k * s.B + b] * expf(mk - m);
        }
        const float lt = s.lt[b];
        const float D = __fmaf_rn(s.w, z, expf(lt - m));
        s.row_m[b] = m;
        s.row_inv[b] = 1.f / D;
        loss = s.weight * ((m + logf(D)) - lt);
    }
    loss = warp_sum(loss);
    if ((threadIdx.x & 31) == 0 && s.loss) atomicAdd(s.loss, (double)loss);
}

// The per-element rules of the dQ and dX passes.  Each pass calls, per CTA and tile:
//   dq_begin(q0, first entity of the split)   once, before the dQ pass's first entity tile;
//   dq_tile(e0) / dx_tile(q0, e0)             before the tile's ova_logits (whose barriers publish what it writes);
//   grad<LOSS>(acc, b, i, c, e)               dL/dl of row b = q0 + 2 ty + i (the thread's i-th row) and entity
//                                             e = e0 + c, zero outside the batch or past n_ent; LOSS (dQ only) also
//                                             adds the element's loss to the thread's partial sum;
//   dq_end()                                  once, after the dQ pass.
// 1vsAll: the multiclass rule, with each row's target, max and 1 / D from the merge pass.
struct OvaMulticlass {
    const OneVsAllSide &s;
    long long tgt[2];
    float m[2], inv[2];
    __device__ __forceinline__ OvaMulticlass(const OneVsAllSide &s_, float *) : s(s_) {}
    __device__ __forceinline__ void rows(long long q0, int tid)
    {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const long long b = q0 + 2 * (tid >> 4) + i;
            tgt[i] = b < s.B ? s.triples[3 * b + s.col] : -1;
            m[i] = b < s.B ? s.row_m[b] : 0.f;
            inv[i] = b < s.B ? s.row_inv[b] : 0.f;
        }
    }
    __device__ __forceinline__ void dq_begin(long long q0, long long, int tid) { rows(q0, tid); }
    __device__ __forceinline__ void dq_tile(long long, int) {}
    __device__ __forceinline__ void dx_tile(long long q0, long long, int tid) { rows(q0, tid); }
    template <bool LOSS>
    __device__ __forceinline__ float grad(float acc, long long, int i, int, long long e)
    {
        return (tgt[i] >= 0 && e < s.n_cand) ? ova_grad(acc, s, e, tgt[i], m[i], inv[i]) : 0.f;
    }
    __device__ __forceinline__ void dq_end() {}
};

// KvsAll: the multi-label rule.  Thread r < 32 keeps row q0 + r's cursor into its label slice and writes the row's
// mask of the current entity tile (bit c: entity e0 + c is a label) to shared memory.
struct KvaMultiLabel {
    const OneVsAllSide &s;
    unsigned *mask;       // [32] in shared memory
    long long cur, end;   // thread r < 32: next label of row q0 + r not yet in a mask, and the end of its slice
    float loss;           // the thread's partial loss (dQ)
    __device__ __forceinline__ KvaMultiLabel(const OneVsAllSide &s_, float *mask_)
        : s(s_), mask(reinterpret_cast<unsigned *>(mask_)), cur(0), end(0), loss(0.f) {}
    // thread r < 32: the cursor of row q0 + r at its first label >= e (lower_bound over the ascending slice)
    __device__ __forceinline__ void seek(long long q0, long long e, int tid)
    {
        if (tid >= OVA_T) return;
        const long long b = q0 + tid;
        cur = end = 0;
        if (b >= s.B) return;
        long long lo = s.label_off[b], hi = s.label_off[b + 1];
        end = hi;
        while (lo < hi) {
            const long long mid = (lo + hi) >> 1;
            if (s.label_ids[mid] < e) lo = mid + 1;
            else hi = mid;
        }
        cur = lo;
    }
    // thread r < 32: the labels of row q0 + r in [e0, e0 + 32) -> mask[r]; the cursor moves past them
    __device__ __forceinline__ void build(long long e0, int tid)
    {
        if (tid >= OVA_T) return;
        unsigned bits = 0;
        for (; cur < end; ++cur) {
            const long long d = s.label_ids[cur] - e0;
            if (d >= OVA_T) break;
            bits |= 1u << d;
        }
        mask[tid] = bits;
    }
    __device__ __forceinline__ void dq_begin(long long q0, long long e_first, int tid) { seek(q0, e_first, tid); }
    __device__ __forceinline__ void dq_tile(long long e0, int tid) { build(e0, tid); }
    __device__ __forceinline__ void dx_tile(long long q0, long long e0, int tid)
    {
        seek(q0, e0, tid);
        build(e0, tid);
    }
    template <bool LOSS>
    __device__ __forceinline__ float grad(float acc, long long b, int i, int c, long long e)
    {
        if (b >= s.B || e >= s.n_cand) return 0.f;
        const int r = 2 * (threadIdx.x >> 4) + i;
        const float y = (mask[r] >> c) & 1u ? s.y0 + s.y1 : s.y0;
        bool in;
        const float l = ova_clip(acc, s.scale, in);
        const float z = expf(-fabsf(l));  // e^-|l| <= 1: neither the sigmoid nor the softplus can overflow
        if (LOSS) loss += (fmaxf(l, 0.f) - y * l) + log1pf(z);
        if (!in) return 0.f;
        const float r1 = 1.f / (1.f + z);
        return s.w * ((l >= 0.f ? r1 : z * r1) - y);
    }
    __device__ __forceinline__ void dq_end()
    {
        const float t = warp_sum(loss);
        if ((threadIdx.x & 31) == 0 && s.loss) atomicAdd(s.loss, (double)(s.w * t));
    }
};

// dQ (query tile x entity split).  Shared memory: stage, g tile, [32, ld] accumulator, then the rule's [32] masks.
template <class Rule>
__global__ void __launch_bounds__(OVA_THREADS) kge_ova_dq_kernel(const OneVsAllSide s)
{
    extern __shared__ __align__(16) float ova_sm[];
    float *stage = ova_sm, *gs = ova_sm + OVA_STAGE, *acc_s = gs + OVA_GS;
    const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15, split = blockIdx.y;
    const long long q0 = (long long)blockIdx.x * OVA_T;
    long long et0, et1;
    ova_split_range(s, split, et0, et1);
    ova_zero(acc_s, OVA_T * s.ld, tid);
    Rule rule(s, acc_s + (size_t)OVA_T * s.ld);
    rule.dq_begin(q0, et0 * OVA_T, tid);
    for (long long et = et0; et < et1; ++et) {
        const long long e0 = et * OVA_T;
        rule.dq_tile(e0, tid);
        float acc[2][2];
        ova_logits(s.q, q0, s.B, s.cand, e0, s.n_cand, s.ld, stage, tid, acc);
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const long long e = e0 + tx + 16 * j;
                gs[(2 * ty + i) * (OVA_T + 1) + tx + 16 * j] =
                    rule.template grad<true>(acc[i][j], q0 + 2 * ty + i, i, tx + 16 * j, e);
            }
        __syncthreads();
        ova_accumulate<false>(acc_s, gs, s.cand, e0, s.n_cand, s.ld, stage, tid);
    }
    rule.dq_end();
    // this split's partial Gq rows, scale included
    const int o = tid >> 3;
    const long long b = q0 + o;
    if (b < s.B)
        for (int c = (tid & 7) * 4; c < s.ld; c += 32) {
            const float4 a = ova_lds4(acc_s + (size_t)o * s.ld + c);
            *reinterpret_cast<float4 *>(s.pgq + ((size_t)split * s.B + b) * s.ld + c) = s.scale * a;
        }
}

// dX (candidate tile x query-tile split: every query tile when s.xsplit = 1); the same shared memory as dQ
template <class Rule>
__global__ void __launch_bounds__(OVA_THREADS) kge_ova_dx_kernel(const OneVsAllSide s)
{
    extern __shared__ __align__(16) float ova_sm[];
    float *stage = ova_sm, *gs = ova_sm + OVA_STAGE, *acc_s = gs + OVA_GS;
    const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15, split = blockIdx.y;
    const long long e0 = (long long)blockIdx.x * OVA_T;
    ova_zero(acc_s, OVA_T * s.ld, tid);
    Rule rule(s, acc_s + (size_t)OVA_T * s.ld);
    const long long n_qt = (s.B + OVA_T - 1) / OVA_T;
    for (long long qt = split; qt < n_qt; qt += s.xsplit) {  // split k takes the query tiles k, k + xsplit, ...
        const long long q0 = qt * OVA_T;
        rule.dx_tile(q0, e0, tid);
        float acc[2][2];
        ova_logits(s.q, q0, s.B, s.cand, e0, s.n_cand, s.ld, stage, tid, acc);
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                const long long e = e0 + tx + 16 * j;
                gs[(2 * ty + i) * (OVA_T + 1) + tx + 16 * j] =
                    rule.template grad<false>(acc[i][j], q0 + 2 * ty + i, i, tx + 16 * j, e);
            }
        __syncthreads();
        ova_accumulate<true>(acc_s, gs, s.q, q0, s.B, s.ld, stage, tid);
    }
    // one add per gradient row: this CTA is the only writer of its rows in this launch (split: of its partial rows)
    const int o = tid >> 3;
    const long long e = e0 + o;
    if (e < s.n_cand)
        for (int c = (tid & 7) * 4; c < s.ld; c += 32) {
            const float4 a = ova_lds4(acc_s + (size_t)o * s.ld + c);
            if (s.xsplit == 1) {
                float *g = s.grad_cand + (size_t)e * s.ld + c;
                *reinterpret_cast<float4 *>(g) = *reinterpret_cast<const float4 *>(g) + s.scale * a;
            } else {
                *reinterpret_cast<float4 *>(s.pgx + ((size_t)split * s.n_cand + e) * s.ld + c) = s.scale * a;
            }
        }
}

// grad_cand[e] += sum of the xsplit partial dX rows of e, in split order (one thread per float4: one writer per row)
__global__ void __launch_bounds__(256) kge_ova_dx_sum_kernel(const OneVsAllSide s)
{
    const int nq4 = s.ld / 4;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= s.n_cand * nq4) return;
    const size_t off = (size_t)idx * 4;  // = e * ld + 4 * chunk
    float4 a = f4ld(s.pgx + off);
    for (int k = 1; k < s.xsplit; ++k) a = a + f4ld(s.pgx + (size_t)k * s.n_cand * s.ld + off);
    f4st(s.grad_cand + off, f4ld(s.grad_cand + off) + a);
}

// one thread per (positive, float4 chunk of a half).  REL: the relation side, whose query is Qp(s, o) = d f / dp, so
// by linearity in the relation row d/ds = Q0(Gq, o) and d/do = Q1(s, Gq), with Gq in the relation slot.
template <int HALVES, bool REL>
__global__ void __launch_bounds__(256) kge_ova_chain_kernel(const OneVsAllSide s)
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
    if constexpr (REL) {
        const float *srow = s.ent + (size_t)si * s.ld, *orow = s.ent + (size_t)oi_ * s.ld;
        const float4 sr = f4ld(srow + d), sim = HALVES == 2 ? f4ld(srow + di) : f4zero();
        const float4 orr = f4ld(orow + d), oim = HALVES == 2 ? f4ld(orow + di) : f4zero();
        float *gs_ = s.grad_ent + (size_t)si * s.ld, *go = s.grad_ent + (size_t)oi_ * s.ld;
        red_add_v4(gs_ + d, query_subj<HALVES, 0>(Gr, Gi, orr, oim));
        red_add_v4(go + d, query_obj<HALVES, 0>(sr, sim, Gr, Gi));
        if (HALVES == 2) {
            red_add_v4(gs_ + di, query_subj<HALVES, 1>(Gr, Gi, orr, oim));
            red_add_v4(go + di, query_obj<HALVES, 1>(sr, sim, Gr, Gi));
        }
        if (d == 0 && s.stamp_ent) {
            s.stamp_ent[si] = s.stamp;
            s.stamp_ent[oi_] = s.stamp;
        }
        return;
    }
    const float *prow = s.rel + (size_t)pi_ * s.ld;
    const float4 pr = f4ld(prow + d), pi = HALVES == 2 ? f4ld(prow + di) : f4zero();
    const float4 z = f4zero();
    float *gp = s.grad_rel + (size_t)pi_ * s.ld;
    if (s.side == KGE_SIDE_O) {  // q = Q1(s, p): d/ds = Q0(p, Gq), d/dp of f(s, p, Gq)
        const float *srow = s.ent + (size_t)si * s.ld;
        const float4 sr = f4ld(srow + d), sim = HALVES == 2 ? f4ld(srow + di) : f4zero();
        float *ge = s.grad_ent + (size_t)si * s.ld;
        red_add_v4(ge + d, query_subj<HALVES, 0>(pr, pi, Gr, Gi));
        red_add_v4(gp + d, trilinear_grad_p<HALVES, 0>(sr, sim, z, z, z, z, Gr, Gi));
        if (HALVES == 2) {
            red_add_v4(ge + di, query_subj<HALVES, 1>(pr, pi, Gr, Gi));
            red_add_v4(gp + di, trilinear_grad_p<HALVES, 1>(sr, sim, z, z, z, z, Gr, Gi));
        }
    } else {  // q = Q0(p, o): d/do = Q1(Gq, p), d/dp of f(Gq, p, o)
        const float *orow = s.ent + (size_t)oi_ * s.ld;
        const float4 orr = f4ld(orow + d), oim = HALVES == 2 ? f4ld(orow + di) : f4zero();
        float *ge = s.grad_ent + (size_t)oi_ * s.ld;
        red_add_v4(ge + d, query_obj<HALVES, 0>(Gr, Gi, pr, pi));
        red_add_v4(gp + d, trilinear_grad_p<HALVES, 0>(z, z, orr, oim, Gr, Gi, z, z));
        if (HALVES == 2) {
            red_add_v4(ge + di, query_obj<HALVES, 1>(Gr, Gi, pr, pi));
            red_add_v4(gp + di, trilinear_grad_p<HALVES, 1>(z, z, orr, oim, Gr, Gi, z, z));
        }
    }
    if (d == 0 && s.stamp_rel) s.stamp_rel[pi_] = s.stamp;
}

__global__ void kge_ova_stamp_kernel(int *stamps, long long n, int stamp)
{
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        stamps[i] = stamp;
}

// the dQ, dX and chain passes of one side under the per-element rule Rule (smem: dynamic bytes of dQ and dX)
template <class Rule>
static cudaError_t launch_grad_passes(const OneVsAllSide &s, int halves, size_t smem, cudaStream_t st,
                                      const SideDropout *drop)
{
    const unsigned n_qt = (unsigned)((s.B + OVA_T - 1) / OVA_T), n_et = (unsigned)((s.n_cand + OVA_T - 1) / OVA_T);
    cudaError_t e;
    if ((e = launch_with_smem(kge_ova_dq_kernel<Rule>, dim3(n_qt, s.nsplit), OVA_THREADS, smem, st, s)) != cudaSuccess) return e;
    if ((e = launch_with_smem(kge_ova_dx_kernel<Rule>, dim3(n_et, s.xsplit), OVA_THREADS, smem, st, s)) != cudaSuccess)
        return e;
    if (s.xsplit > 1) {
        kge_ova_dx_sum_kernel<<<(unsigned)((s.n_cand * (s.ld / 4) + 255) / 256), 256, 0, st>>>(s);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
    }
    if (drop) return launch_dropout_finish(s, *drop, halves, st);  // masked candidate rows, then the dropout chain pass
    const unsigned grid = (unsigned)((s.B * (s.kp / 4) + 255) / 256);
    const bool rel = s.side == KGE_SIDE_P;
    if (halves == 2) {
        if (rel) kge_ova_chain_kernel<2, true><<<grid, 256, 0, st>>>(s);
        else kge_ova_chain_kernel<2, false><<<grid, 256, 0, st>>>(s);
    } else {
        if (rel) kge_ova_chain_kernel<1, true><<<grid, 256, 0, st>>>(s);
        else kge_ova_chain_kernel<1, false><<<grid, 256, 0, st>>>(s);
    }
    return cudaGetLastError();
}

// qp[b] = Qp(s_b, o_b) = d f(s_b, p, o_b) / dp (scale excluded), the relation side's query: one thread per (positive,
// float4 chunk of a half), with the training kernels' relation-row gradient arithmetic (U = s in the subject slot)
template <int HALVES>
__global__ void __launch_bounds__(256) kge_ova_relation_query_kernel(const OneVsAllSide s, float *qp)
{
    const int nq4 = s.kp / 4;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= s.B * nq4) return;
    const long long b = idx / nq4;
    const int d = (int)(idx - b * nq4) * 4, di = HALVES == 2 ? s.kp + d : d;
    const float *srow = s.ent + (size_t)s.triples[3 * b] * s.ld, *orow = s.ent + (size_t)s.triples[3 * b + 2] * s.ld;
    const float4 sr = f4ld(srow + d), sim = HALVES == 2 ? f4ld(srow + di) : f4zero();
    const float4 orr = f4ld(orow + d), oim = HALVES == 2 ? f4ld(orow + di) : f4zero();
    const float4 z = f4zero();
    float *q = qp + (size_t)b * s.ld;
    f4st(q + d, trilinear_grad_p<HALVES, 0>(z, z, orr, oim, sr, sim, z, z));
    if (HALVES == 2) f4st(q + di, trilinear_grad_p<HALVES, 1>(z, z, orr, oim, sr, sim, z, z));
}

// With dropout the side's passes read its dropped candidate table and queries (launch_dropout_prepare)
cudaError_t launch_one_vs_all_side(const OneVsAllSide &s_, int halves, cudaStream_t st, const SideDropout *drop)
{
    if (s_.B == 0) return cudaSuccess;
    OneVsAllSide s = s_;
    cudaError_t e;
    if (drop && (e = launch_dropout_prepare(s, *drop, const_cast<float *>(s.q), halves, st)) != cudaSuccess) return e;
    const unsigned n_qt = (unsigned)((s.B + OVA_T - 1) / OVA_T);
    e = launch_with_smem(kge_ova_stats_kernel, dim3(n_qt, s.nsplit), OVA_THREADS, OVA_STAGE * sizeof(float), st, s);
    if (e != cudaSuccess) return e;
    kge_ova_merge_kernel<<<(unsigned)((s.B + 255) / 256), 256, 0, st>>>(s);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    return launch_grad_passes<OvaMulticlass>(s, halves, one_vs_all_smem_bytes(s.ld), st, drop);
}

cudaError_t launch_relation_prediction_side(const OneVsAllSide &s, float *qp, int halves, cudaStream_t st,
                                            const SideDropout *drop)
{
    if (s.B == 0) return cudaSuccess;
    if (drop) return launch_one_vs_all_side(s, halves, st, drop);  // the queries come from the dropped s and o rows
    const unsigned grid = (unsigned)((s.B * (s.kp / 4) + 255) / 256);
    if (halves == 2) kge_ova_relation_query_kernel<2><<<grid, 256, 0, st>>>(s, qp);
    else kge_ova_relation_query_kernel<1><<<grid, 256, 0, st>>>(s, qp);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    return launch_one_vs_all_side(s, halves, st);
}

size_t k_vs_all_smem_bytes(int ld) { return one_vs_all_smem_bytes(ld) + OVA_T * sizeof(unsigned); }

cudaError_t launch_k_vs_all_side(const OneVsAllSide &s_, int halves, cudaStream_t st, const SideDropout *drop)
{
    if (s_.B == 0) return cudaSuccess;
    OneVsAllSide s = s_;
    cudaError_t e;
    if (drop && (e = launch_dropout_prepare(s, *drop, const_cast<float *>(s.q), halves, st)) != cudaSuccess) return e;
    return launch_grad_passes<KvaMultiLabel>(s, halves, k_vs_all_smem_bytes(s.ld), st, drop);
}

cudaError_t launch_one_vs_all_stamps(int *stamp_ent, long long n_ent, int stamp, cudaStream_t st)
{
    if (!stamp_ent || n_ent == 0) return cudaSuccess;
    const long long blocks = (n_ent + 255) / 256;
    kge_ova_stamp_kernel<<<(unsigned)(blocks < 4096 ? blocks : 4096), 256, 0, st>>>(stamp_ent, n_ent, stamp);
    return cudaGetLastError();
}

}  // namespace kge
