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
// Every g * Q term is bit-identical to the one the scatter path sends; only the order of the fp32 additions differs
// (within a run: entry order; across runs and with the other REDs: atomic order).
#include "kge_train_common.cuh"

namespace kge {

__global__ void kge_bucket_count_kernel(const TrainParams p)
{
    const long long n = (long long)p.eta * p.B;
    for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (long long)gridDim.x * blockDim.x) {
        int keep, repl;
        if (p.neg_ent) repl = p.neg_ent[r];
        else draw_corruption(p.seed, p.step, (unsigned long long)r, p.n_ent, &keep, &repl);
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

template <int HALVES, int NIT>
__global__ void __launch_bounds__(256) kge_bucket_sum_kernel(const TrainParams p)
{
    const int lane = threadIdx.x & 31;
    const long long n = (long long)p.eta * p.B;
    const long long base = ((long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * 32;
    if (base >= n) return;
    const int cnt = (int)min(32ll, n - base);
    const int nch = p.kp >> 2;
    const uint32_t hsB = (uint32_t)p.kp * 4u;
    uint32_t off[NIT];
    bool live[NIT];
#pragma unroll
    for (int it = 0; it < NIT; ++it) {
        const int c = lane + 32 * it;
        live[it] = c < nch;
        off[it] = 16u * (uint32_t)min(c, nch - 1);
    }
    // this run's entries, one per lane, broadcast one at a time below
    int m_e = -1, m_o = 0, m_r = 0;
    float m_g = 0.f;
    if (lane < cnt) {
        m_e = p.bk.eid[base + lane];
        m_o = p.bk.other[base + lane];
        m_r = p.bk.rel[base + lane];
        m_g = p.bk.g[base + lane];
    }
    const char *const ent = reinterpret_cast<const char *>(p.ent);
    const char *const rel = reinterpret_cast<const char *>(p.rel);
    const size_t row_bytes = (size_t)p.ld * 4u;
    float4 ar[NIT], ai[NIT];
#pragma unroll
    for (int it = 0; it < NIT; ++it) ar[it] = ai[it] = f4zero();
    int cur = __shfl_sync(0xffffffffu, m_e, 0);
    auto flush = [&]() {
        char *const g0 = reinterpret_cast<char *>(p.grad_ent) + (size_t)cur * row_bytes;
#pragma unroll
        for (int it = 0; it < NIT; ++it) {
            if (!live[it]) continue;
            red4(g0, off[it], ar[it]);
            if constexpr (HALVES == 2) red4(g0, off[it] + hsB, ai[it]);
            ar[it] = ai[it] = f4zero();
        }
    };
    // two entries per trip: both entries' rows are requested before either is used
    for (int k = 0; k < cnt; k += 2) {
        const bool has_b = k + 1 < cnt;
        const int kb = has_b ? k + 1 : k;
        const int ea = __shfl_sync(0xffffffffu, m_e, k), eb = __shfl_sync(0xffffffffu, m_e, kb);
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
        auto add = [&](int e, int r, float g, const float4(&xr)[NIT], const float4(&xi)[NIT], const float4(&pr)[NIT],
                       const float4(&pi)[NIT]) {
            if (e != cur) {
                flush();
                cur = e;
            }
#pragma unroll
            for (int it = 0; it < NIT; ++it) {
                float4 qr, qi = f4zero();
                if (r < 0) query_obj<HALVES>(xr[it], xi[it], pr[it], pi[it], qr, qi);  // object replaced: x is the subject
                else query_subj<HALVES>(pr[it], pi[it], xr[it], xi[it], qr, qi);      // subject replaced: x is the object
                ar[it] = ar[it] + g * qr;
                if constexpr (HALVES == 2) ai[it] = ai[it] + g * qi;
            }
        };
        add(ea, ra, ga, xar, xai, par, pai);
        if (has_b) add(eb, rb, gb, xbr, xbi, pbr, pbi);
    }
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

template <int HALVES, int NIT>
static cudaError_t launch_sum(const TrainParams &p, cudaStream_t st)
{
    const long long runs = ((long long)p.eta * p.B + 31) / 32;
    kge_bucket_sum_kernel<HALVES, NIT><<<(int)((runs + 7) / 8), 256, 0, st>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_bucket_sum(const TrainParams &p, int nit, cudaStream_t st)
{
    if (p.B == 0) return cudaSuccess;
    const bool two = p.model != KGE_DISTMULT;
    if (nit <= 1) return two ? launch_sum<2, 1>(p, st) : launch_sum<1, 1>(p, st);
    if (nit == 2) return two ? launch_sum<2, 2>(p, st) : launch_sum<1, 2>(p, st);
    if (two) return cudaErrorInvalidValue;
    return launch_sum<1, 4>(p, st);
}

}  // namespace kge
