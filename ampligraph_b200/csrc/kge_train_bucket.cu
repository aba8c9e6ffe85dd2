// kge_train_bucket.cu -- owner-computes gradient rows of the replaced entities for the resident fast path (sm_90a).
//
// In the fused kernel every corruption adds g * Q (kge_train_common.cuh: query_subj / query_obj) to its replaced
// entity's gradient row.  Replaced entities are drawn uniformly, so those adds are eta*B full-row REDs to uniformly
// random rows (cfg2: 272,120 per step, three quarters of the kernel's RED bytes) with no reuse inside a CTA to combine
// them.  Here the sum changes hands instead:
//   1. kge_bucket_count_kernel: each corruption r = j*B+i draws (keep, repl) exactly as the fused kernel will and takes a
//      rank in repl's bucket (one integer atomic per corruption).
//   2. kge_bucket_tile_sum_kernel + kge_bucket_scan_kernel: a two-level scan, one CTA per 8,192 entities, turns the
//      per-entity counts into CSR offsets and zeroes the counts again, so the next step needs no memset.
//   3. The fused kernel, GATHER instantiation (kge_train_res.cu), writes each corruption's g, entity, kept-side entity and
//      relation | side at offset[repl] + rank instead of issuing its REDs.
//   4. kge_bucket_sum_kernel: one warp per run of 32 consecutive entries (each entity's entries are contiguous, so a run
//      covers a few whole buckets, or part of a long one) re-forms Q from the kept-side entity row and the relation row
//      with the fused kernel's operations, accumulates g * Q in registers in entry order, and adds the sum to the
//      gradient row with one set of REDs per entity and run.  A RED rather than a store, so that a bucket split over
//      two runs, and the s / o rows the fused kernel scatters into the same table, add up without ordering.
//   5. Or, for a step run with KGE_STEP_FUSED_DEFER, step 4 waits for kge_optimizer_step_deferred, whose kernel
//      (kge_bucket_owner_kernel) gives each row of the [ent | rel] block to one warp: it sums the row's whole bucket in
//      entry order, adds it to the row's gradient and applies the dense optimizer, reading the parameter block the step
//      trained on and writing the new rows to a second block.  The bucket sum's row reads are latency bound and the
//      optimizer's streams are HBM bound, so in one kernel each runs under the other (DESIGN.md 3.2).
// Every g * Q term is bit-identical to the one the scatter path sends; only the order of the fp32 additions differs
// (within a run: entry order; across runs and with the other REDs: atomic order).
#include "kge_optim_common.cuh"
#include "kge_train_common.cuh"

namespace kge {

__global__ void kge_bucket_count_kernel(const TrainParams p)
{
    const long long n = (long long)p.eta * p.B;
    for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (long long)gridDim.x * blockDim.x) {
        int keep, repl;
        corruption_of(p, (unsigned long long)r, keep, repl);
        p.bk.pos[r] = atomicAdd(p.bk.cnt + repl, 1);
    }
}

// Two-level scan over the per-entity counts, one CTA per tile of KGE_SCAN_TILE entities, so its cost does not grow with
// n_ent on one SM: kge_bucket_tile_sum_kernel writes each tile's total, kge_bucket_scan_kernel sums the totals of the tiles
// before its own and scans its tile.  Every global access is coalesced: a tile's counts are staged in shared memory and
// each thread scans 8 consecutive ones there.  (With each thread reading its own consecutive counts from global memory,
// one SM spent ~25 us per 16 K counts on H100; a single CTA walking all tiles spent ~4 us per tile.)
#define KGE_SCAN_THREADS 1024
#define KGE_SCAN_ITEMS 8
#define KGE_SCAN_TILE (KGE_SCAN_THREADS * KGE_SCAN_ITEMS)

// sum of v over the CTA, returned to every thread; red: KGE_SCAN_THREADS / 32 ints of shared memory
__device__ __forceinline__ int block_sum(int v, int *red)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    v = __reduce_add_sync(0xffffffffu, v);
    if (lane == 0) red[warp] = v;
    __syncthreads();
    v = __reduce_add_sync(0xffffffffu, red[lane]);
    __syncthreads();  // red may be reused
    return v;
}

__global__ void __launch_bounds__(KGE_SCAN_THREADS) kge_bucket_tile_sum_kernel(const int *cnt, int *tiles, int n_ent)
{
    __shared__ int red[KGE_SCAN_THREADS / 32];
    const int base = blockIdx.x * KGE_SCAN_TILE;
    int s = 0;
#pragma unroll
    for (int q = 0; q < KGE_SCAN_ITEMS; ++q) {
        const int e = base + q * KGE_SCAN_THREADS + threadIdx.x;
        if (e < n_ent) s += cnt[e];
    }
    s = block_sum(s, red);
    if (threadIdx.x == 0) tiles[blockIdx.x] = s;
}

__global__ void __launch_bounds__(KGE_SCAN_THREADS) kge_bucket_scan_kernel(int *cnt, int *off, const int *tiles, int n_ent)
{
    __shared__ int buf[KGE_SCAN_TILE];
    __shared__ int warp_tot[KGE_SCAN_THREADS / 32];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const int base = blockIdx.x * KGE_SCAN_TILE;
    int carry = 0;  // entries of the tiles before this one
    for (int j = t; j < (int)blockIdx.x; j += KGE_SCAN_THREADS) carry += tiles[j];
    carry = block_sum(carry, warp_tot);
#pragma unroll
    for (int q = 0; q < KGE_SCAN_ITEMS; ++q) {
        const int e = base + q * KGE_SCAN_THREADS + t;
        buf[q * KGE_SCAN_THREADS + t] = e < n_ent ? cnt[e] : 0;
        if (e < n_ent) cnt[e] = 0;  // ready for the next step's count
    }
    __syncthreads();
    int c[KGE_SCAN_ITEMS], s = 0;
#pragma unroll
    for (int q = 0; q < KGE_SCAN_ITEMS; ++q) s += (c[q] = buf[t * KGE_SCAN_ITEMS + q]);
    int x = s;  // inclusive warp scan
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= d) x += y;
    }
    if (lane == 31) warp_tot[warp] = x;
    __syncthreads();
    if (warp == 0) {
        int w = warp_tot[lane];
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, w, d);
            if (lane >= d) w += y;
        }
        warp_tot[lane] = w;  // inclusive over warps
    }
    __syncthreads();
    int run = carry + x - s + (warp ? warp_tot[warp - 1] : 0);
#pragma unroll
    for (int q = 0; q < KGE_SCAN_ITEMS; ++q) {
        buf[t * KGE_SCAN_ITEMS + q] = run;
        run += c[q];
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < KGE_SCAN_ITEMS; ++q) {
        const int e = base + q * KGE_SCAN_THREADS + t;
        if (e < n_ent) off[e] = buf[q * KGE_SCAN_THREADS + t];
    }
    if (blockIdx.x == gridDim.x - 1 && t == 0) off[n_ent] = carry + warp_tot[KGE_SCAN_THREADS / 32 - 1];
}

// A lane's share of a row of the parameter, gradient and slot tables: float4 chunk c = lane + 32 * it of each half sits
// at byte offset off[it] (+ hsB for the im half).  live[it] is false past the row's kp / 4 chunks; there off[it] repeats
// the last chunk, so that loads stay inside the row, and the result is dropped.
template <int NIT>
struct LaneRow {
    uint32_t off[NIT];
    bool live[NIT];
    uint32_t hsB;
    size_t row_bytes;
    __device__ __forceinline__ LaneRow(const TrainParams &p, int lane)
    {
        const int nch = p.kp >> 2;
        hsB = (uint32_t)p.kp * 4u;
        row_bytes = (size_t)p.ld * 4u;
#pragma unroll
        for (int it = 0; it < NIT; ++it) {
            const int c = lane + 32 * it;
            live[it] = c < nch;
            off[it] = 16u * (uint32_t)min(c, nch - 1);
        }
    }
};

// The bucket walk of both replaced-row sums: adds g * Q of the cnt <= 32 bucket entries from base on to the lane's chunks
// ar / ai (re / im halves) in entry order.  Q is re-formed from the kept-side entity row and the relation row with the
// fused kernel's operations.  The entries are read one per lane and broadcast, two per trip, so that both entries' rows
// are requested before either is used.  Lane k's key goes with entry base + k: before_add(key) runs before the entry is
// added (kge_bucket_sum_kernel passes the entity and flushes its sum when that changes).
template <int HALVES, int NIT, class Index, class Hook>
__device__ __forceinline__ void bucket_walk(const TrainParams &p, const LaneRow<NIT> &w, Index base, int cnt, int key,
                                            float4 (&ar)[NIT], float4 (&ai)[NIT], Hook &&before_add)
{
    const int lane = threadIdx.x & 31;
    const uint32_t(&off)[NIT] = w.off;
    const uint32_t hsB = w.hsB;
    const size_t row_bytes = w.row_bytes;
    const char *const ent = reinterpret_cast<const char *>(p.ent);
    const char *const rel = reinterpret_cast<const char *>(p.rel);
    int m_o = 0, m_r = 0;
    float m_g = 0.f;
    if (lane < cnt) {
        m_o = p.bk.other[base + lane];
        m_r = p.bk.rel[base + lane];
        m_g = p.bk.g[base + lane];
    }
    for (int k = 0; k < cnt; k += 2) {
        const bool has_b = k + 1 < cnt;
        const int kb = has_b ? k + 1 : k;
        const int key_a = __shfl_sync(0xffffffffu, key, k), key_b = __shfl_sync(0xffffffffu, key, kb);
        const int oa = __shfl_sync(0xffffffffu, m_o, k), ob = __shfl_sync(0xffffffffu, m_o, kb);
        const int ra = __shfl_sync(0xffffffffu, m_r, k), rb = __shfl_sync(0xffffffffu, m_r, kb);
        const float ga = __shfl_sync(0xffffffffu, m_g, k), gb = __shfl_sync(0xffffffffu, m_g, kb);
        const char *const xa = ent + (size_t)oa * row_bytes, *const xb = ent + (size_t)ob * row_bytes;
        const char *const pa = rel + (size_t)(ra & 0x7fffffff) * row_bytes, *const pb = rel + (size_t)(rb & 0x7fffffff) * row_bytes;
        float4 xar[NIT], xai[NIT], xbr[NIT], xbi[NIT], par[NIT], pai[NIT], pbr[NIT], pbi[NIT];
#pragma unroll
        for (int it = 0; it < NIT; ++it) {
            xar[it] = __ldg(reinterpret_cast<const float4 *>(xa + off[it]));
            xbr[it] = __ldg(reinterpret_cast<const float4 *>(xb + off[it]));
            par[it] = __ldg(reinterpret_cast<const float4 *>(pa + off[it]));
            pbr[it] = __ldg(reinterpret_cast<const float4 *>(pb + off[it]));
            if constexpr (HALVES == 2) {
                xai[it] = __ldg(reinterpret_cast<const float4 *>(xa + off[it] + hsB));
                xbi[it] = __ldg(reinterpret_cast<const float4 *>(xb + off[it] + hsB));
                pai[it] = __ldg(reinterpret_cast<const float4 *>(pa + off[it] + hsB));
                pbi[it] = __ldg(reinterpret_cast<const float4 *>(pb + off[it] + hsB));
            } else {
                xai[it] = xbi[it] = pai[it] = pbi[it] = f4zero();
            }
        }
        auto add = [&](int r, float g, const float4(&xr)[NIT], const float4(&xi)[NIT], const float4(&pr)[NIT],
                       const float4(&pi)[NIT]) {
#pragma unroll
            for (int it = 0; it < NIT; ++it) {
                float4 qr, qi = f4zero();
                if (r < 0) query_obj<HALVES>(xr[it], xi[it], pr[it], pi[it], qr, qi);  // object replaced: x is the subject
                else query_subj<HALVES>(pr[it], pi[it], xr[it], xi[it], qr, qi);      // subject replaced: x is the object
                ar[it] = ar[it] + g * qr;
                if constexpr (HALVES == 2) ai[it] = ai[it] + g * qi;
            }
        };
        before_add(key_a);
        add(ra, ga, xar, xai, par, pai);
        if (has_b) {
            before_add(key_b);
            add(rb, gb, xbr, xbi, pbr, pbi);
        }
    }
}

template <int HALVES, int NIT>
__global__ void __launch_bounds__(256) kge_bucket_sum_kernel(const TrainParams p)
{
    const int lane = threadIdx.x & 31;
    const long long n = (long long)p.eta * p.B;
    const long long base = ((long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * 32;
    if (base >= n) return;
    const int cnt = (int)min(32ll, n - base);
    const LaneRow<NIT> w(p, lane);
    const int m_e = lane < cnt ? p.bk.eid[base + lane] : -1;  // this run's entities, one per lane
    float4 ar[NIT], ai[NIT];
#pragma unroll
    for (int it = 0; it < NIT; ++it) ar[it] = ai[it] = f4zero();
    int cur = __shfl_sync(0xffffffffu, m_e, 0);
    auto flush = [&]() {
        char *const g0 = reinterpret_cast<char *>(p.grad_ent) + (size_t)cur * w.row_bytes;
#pragma unroll
        for (int it = 0; it < NIT; ++it) {
            if (!w.live[it]) continue;
            red4(g0, w.off[it], ar[it]);
            if constexpr (HALVES == 2) red4(g0, w.off[it] + w.hsB, ai[it]);
            ar[it] = ai[it] = f4zero();
        }
    };
    bucket_walk<HALVES>(p, w, base, cnt, m_e, ar, ai, [&](int e) {
        if (e != cur) {
            flush();
            cur = e;
        }
    });
    flush();
}

cudaError_t launch_bucket_prepass(const TrainParams &p, cudaStream_t st)
{
    const long long n = (long long)p.eta * p.B;
    const long long blocks = (n + 255) / 256;
    kge_bucket_count_kernel<<<(int)(blocks < 4096 ? blocks : 4096), 256, 0, st>>>(p);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    const int tiles = (int)(((long long)p.n_ent + KGE_SCAN_TILE - 1) / KGE_SCAN_TILE);
    kge_bucket_tile_sum_kernel<<<tiles, KGE_SCAN_THREADS, 0, st>>>(p.bk.cnt, p.bk.tiles, (int)p.n_ent);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    kge_bucket_scan_kernel<<<tiles, KGE_SCAN_THREADS, 0, st>>>(p.bk.cnt, p.bk.off, p.bk.tiles, (int)p.n_ent);
    return cudaGetLastError();
}

cudaError_t launch_bucket_sum(const TrainParams &p, int nit, cudaStream_t st)
{
    if (p.B == 0) return cudaSuccess;
    const long long runs = ((long long)p.eta * p.B + 31) / 32;
    return dispatch_trilinear_shape(p.model, nit, [&](auto halves, auto nits) {
        kge_bucket_sum_kernel<halves, nits><<<(int)((runs + 7) / 8), 256, 0, st>>>(p);
        return cudaGetLastError();
    });
}

// kge_optimizer_step_deferred: one warp per row e of the [ent | rel] block, the row's OWNER.  It walks e's bucket
// [off[e], off[e+1]) in entry order (relation rows and entities nobody replaced have none), re-forms each entry's Q from
// the kept-side entity row and the relation row with the fused kernel's operations and sums g * Q in registers; then the
// dense optimizer: g = grad[e] + sum (in that order; grad[e] holds the fused kernel's s / o / relation REDs), the update4 of
// kge_optim_common.cuh, the new row to the SECOND block x.out, m / v in place, grad[e] = 0.  Every row is updated, so the
// dense semantics hold (empty buckets and relation rows still decay m / v and take the regulariser).
// Hazards: the bucket walk and the epilogue read only x.in (p.ent / p.rel are its parts), which nothing writes during the
// kernel, so no warp sees another's new row; row e of grad, slots and x.out has this one writer, so plain loads / stores.
struct OwnerOptim {
    const float *in;  // [rows, ld] parameter block the step read (p.ent and p.rel are its two parts)
    float *out;       // [rows, ld] parameter block written, every column of every row
    float *grad;      // [rows, ld] gradient block (p.grad_ent and p.grad_rel are its two parts), zeroed
    float *s0, *s1;
    long long rows;
    double *reg_loss;
    OptimParams o;
};

__device__ __forceinline__ void prefetch_l2(const void *p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

// Warps (rows) per CTA.  A CTA retires when its longest bucket is walked, and bucket lengths vary (cfg2: about 19
// entries on average), so every warp of a CTA would wait for the slowest: one-warp CTAs free each row's slot as soon as
// that row is done.  With the regulariser each CTA adds its loss with one fp64 atomic to a single address, so those
// steps keep eight rows per CTA rather than issue one such atomic per row.
__host__ __device__ constexpr int owner_warps(bool reg) { return reg ? 8 : 1; }

// -DKGE_PROFILE_OWNER_WALKONLY builds a profiling variant that walks the buckets but drops the epilogue's prefetches,
// loads and stores; -DKGE_PROFILE_OWNER_NOWALK one that runs the epilogue on empty sums.  Together they attribute the
// kernel's time to its two halves (DESIGN.md 5).  The default build sets neither.
template <int HALVES, int NIT, int KIND, bool REG>
__global__ void __launch_bounds__(32 * owner_warps(REG), 16 / owner_warps(REG)) kge_bucket_owner_kernel(const TrainParams p, const OwnerOptim x,
                                                                                                             const OptimStep os)
{
    const bool S0 = uses_slot0(KIND, x.o.momentum), S1 = uses_slot1(KIND, x.o.momentum, x.o.centered);
    const int lane = threadIdx.x & 31;
    const long long e = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    float racc = 0.f;
    if (e < x.rows) {
        const LaneRow<NIT> w(p, lane);
        const size_t row_bytes = w.row_bytes, roff = (size_t)e * row_bytes;
#ifndef KGE_PROFILE_OWNER_WALKONLY
        {
            // the epilogue's HBM streams are requested now, so that their latency runs under the bucket walk: one lane per
            // 128-byte line of the row (at most 17 lines for the 2 KB rows of NIT <= 4), into L2 rather than registers
            const size_t line0 = roff & ~(size_t)127, span = roff + row_bytes - line0;
            if ((size_t)lane * 128u < span) {
                const size_t a = line0 + (size_t)lane * 128u;
                prefetch_l2(reinterpret_cast<const char *>(x.in) + a);
                prefetch_l2(reinterpret_cast<const char *>(x.grad) + a);
                if (S0) prefetch_l2(reinterpret_cast<const char *>(x.s0) + a);
                if (S1) prefetch_l2(reinterpret_cast<const char *>(x.s1) + a);
            }
        }
#endif
#ifdef KGE_PROFILE_OWNER_NOWALK
        const bool ent_row = false;
#else
        const bool ent_row = e < (long long)p.n_ent;
#endif
        const int b0 = ent_row ? p.bk.off[e] : 0, b1 = ent_row ? p.bk.off[e + 1] : 0;
        float4 ar[NIT], ai[NIT];
#pragma unroll
        for (int it = 0; it < NIT; ++it) ar[it] = ai[it] = f4zero();
        for (int base = b0; base < b1; base += 32) bucket_walk<HALVES>(p, w, base, min(32, b1 - base), 0, ar, ai, [](int) {});
#ifdef KGE_PROFILE_OWNER_WALKONLY
        float keep = 0.f;  // keeps the walk alive: a store no real sum takes
#pragma unroll
        for (int it = 0; it < NIT; ++it) keep += ar[it].x + ar[it].y + ar[it].z + ar[it].w + ai[it].x + ai[it].w;
        if (__float_as_uint(keep) == 0x7fc0deadu) x.out[roff / 4 + lane] = keep;
        if (false)
#endif
        {
            // all loads first (L2 hits after the prefetch), then the updates and the stores (m, v, the new row and the
            // zeroed gradient are not read again this step: evict-first)
            const OptimParams op = x.o;
            const char *const xin = reinterpret_cast<const char *>(x.in) + roff;
            char *const gr = reinterpret_cast<char *>(x.grad) + roff;
            char *const xo = reinterpret_cast<char *>(x.out) + roff;
            char *const m0 = reinterpret_cast<char *>(x.s0) + roff;
            char *const m1 = reinterpret_cast<char *>(x.s1) + roff;
            float4 g4[HALVES][NIT], x4[HALVES][NIT], a4[HALVES][NIT], b4[HALVES][NIT];
#pragma unroll
            for (int h = 0; h < HALVES; ++h)
#pragma unroll
                for (int it = 0; it < NIT; ++it) {
                    g4[h][it] = x4[h][it] = a4[h][it] = b4[h][it] = f4zero();
                    if (!w.live[it]) continue;
                    const uint32_t o = w.off[it] + (h ? w.hsB : 0u);
                    g4[h][it] = __ldcs(reinterpret_cast<const float4 *>(gr + o));
                    x4[h][it] = __ldg(reinterpret_cast<const float4 *>(xin + o));
                    if (S0) a4[h][it] = __ldcs(reinterpret_cast<const float4 *>(m0 + o));
                    if (S1) b4[h][it] = __ldcs(reinterpret_cast<const float4 *>(m1 + o));
                }
#pragma unroll
            for (int h = 0; h < HALVES; ++h)
#pragma unroll
                for (int it = 0; it < NIT; ++it) {
                    if (!w.live[it]) continue;
                    const uint32_t o = w.off[it] + (h ? w.hsB : 0u);
                    const float4 g = g4[h][it] + (h ? ai[it] : ar[it]);
                    const float4 xn = update4<KIND, REG>(x4[h][it], g, a4[h][it], b4[h][it], op, os, op.reg, racc);
                    __stcs(reinterpret_cast<float4 *>(xo + o), xn);
                    if (S0) __stcs(reinterpret_cast<float4 *>(m0 + o), a4[h][it]);
                    if (S1) __stcs(reinterpret_cast<float4 *>(m1 + o), b4[h][it]);
                    __stcs(reinterpret_cast<float4 *>(gr + o), f4zero());
                }
        }
    }
    if (REG && x.reg_loss) flush_reg_loss(racc, x.reg_loss);
}

cudaError_t launch_bucket_sum_optimizer(const TrainParams &p, int nit, const OptimParams &o, const OptimStep &os, const float *in, float *out,
                                        float *grad, float *slot0, float *slot1, long long rows, double *reg_loss,
                                        cudaStream_t st)
{
    if (rows == 0) return cudaSuccess;
    const OwnerOptim x{in, out, grad, slot0, slot1, rows, reg_loss, o};
    return dispatch_optimizer(o.kind, o.reg.p > 0, [&](auto kind, auto reg) {
        constexpr int W = owner_warps(reg);
        return dispatch_trilinear_shape(p.model, nit, [&](auto halves, auto nits) {
            kge_bucket_owner_kernel<halves, nits, decltype(kind)::value, decltype(reg)::value><<<(int)((rows + W - 1) / W), 32 * W, 0, st>>>(p, x, os);
            return cudaGetLastError();
        });
    });
}

}  // namespace kge
