// kge_knn.cu -- exact nearest-neighbour and radius search over the rows of a point matrix (sm_90a).
//
// Replaces the host side of discovery.find_nearest_neighbours (discovery.py:1171-1244, sklearn NearestNeighbors
// .kneighbors) and the radius self-joins of discovery.find_duplicates (:714-982, NearestNeighbors.radius_neighbors).
// The distances are scored chunk by chunk by the ranking pair kernel (kge_rank.cu) with the euclidean chain OP_L2_SUB
// or the manhattan chain OP_L1_SUB, both of which write -d, so that the running top-k of kge_topk.cu keeps the nearest
// points.  This file holds what the two searches add around them: the gather of the query rows, the sign flip of a
// chunk for the farthest points, and the radius count / emit epilogue.
#include <math.h>

#include "kge_internal.h"

namespace kge {

__global__ void kge_knn_gather_kernel(const float4 *__restrict__ points, int ld4, const int32_t *__restrict__ query_ids,
                                      long long b, float4 *__restrict__ qvec)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= b * ld4) return;
    const long long q = i / ld4;
    const int c = (int)(i - q * ld4);
    qvec[i] = points[(size_t)query_ids[q] * ld4 + c];
}

cudaError_t launch_knn_gather(const float *points, int ld, const int32_t *query_ids, long long b, float *qvec, cudaStream_t st)
{
    const long long n = b * (ld / 4);
    if (n == 0) return cudaSuccess;
    kge_knn_gather_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>((const float4 *)points, ld / 4, query_ids, b,
                                                                      (float4 *)qvec);
    return cudaGetLastError();
}

__global__ void kge_knn_negate_kernel(float *__restrict__ x, long long n)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) x[i] = -x[i];
}

cudaError_t launch_knn_negate(float *x, long long n, cudaStream_t st)
{
    if (n == 0) return cudaSuccess;
    kge_knn_negate_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(x, n);
    return cudaGetLastError();
}

// Radius epilogue, one CTA per query row.  The test is -score <= radius, i.e. d <= radius (negation is exact; a NaN
// distance never passes).  Count: every thread counts its columns, one shared atomic per warp.  Emit: the chunk is
// walked in tiles of RN_THREADS columns; a tile's flags are ranked by a block-wide exclusive scan (a ballot per warp,
// then the warp totals), so the hits leave in ascending column order, and the row's cursor -- carried across tiles in a
// register and across chunks in the workspace -- places them after those of the earlier chunks.  No slot is taken by
// an unordered atomic, so the output is deterministic.
constexpr int RN_THREADS = 512, RN_WARPS = RN_THREADS / 32;

template <bool EMIT>
__global__ void __launch_bounds__(RN_THREADS) kge_radius_kernel(const float *__restrict__ chunk, long long ld, long long n,
                                                                long long base, float radius,
                                                                const int32_t *__restrict__ cand_ids, long long cand_begin,
                                                                long long *__restrict__ cursor,
                                                                const long long *__restrict__ off, int32_t *__restrict__ nbr)
{
    __shared__ int warp_tot[RN_WARPS];
    __shared__ int s_cnt;
    const long long q = blockIdx.x;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const float *row = chunk + (size_t)q * ld;
    if (!EMIT) {
        if (t == 0) s_cnt = 0;
        __syncthreads();
        int c = 0;
        for (long long j = t; j < n; j += RN_THREADS) c += (-row[j] <= radius);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
        if (lane == 0 && c) atomicAdd(&s_cnt, c);  // integer sum: order-independent
        __syncthreads();
        if (t == 0) cursor[q] += s_cnt;
        return;
    }
    const long long o0 = off[q], cap = off[q + 1] - o0;
    long long cur = cursor[q];  // CTA-uniform
    for (long long t0 = 0; t0 < n; t0 += RN_THREADS) {
        const long long j = t0 + t;
        const bool hit = j < n && -row[j] <= radius;
        const unsigned m = __ballot_sync(0xffffffffu, hit);
        if (lane == 0) warp_tot[warp] = __popc(m);
        __syncthreads();
        int before = 0, total = 0;
#pragma unroll
        for (int w = 0; w < RN_WARPS; ++w) {
            const int v = warp_tot[w];
            before += w < warp ? v : 0;
            total += v;
        }
        if (hit) {
            const long long at = cur + before + __popc(m & ((1u << lane) - 1u));
            const long long pos = base + j;
            if (at < cap) nbr[o0 + at] = cand_ids ? cand_ids[pos] : (int32_t)(cand_begin + pos);
        }
        cur += total;
        __syncthreads();  // warp_tot is rewritten by the next tile
    }
    if (t == 0) cursor[q] = cur;
}

cudaError_t launch_radius_chunk(const float *chunk, long long ld, long long n, long long base, long long b, float radius,
                                const int32_t *cand_ids, long long cand_begin, long long *cursor, const long long *off,
                                int32_t *nbr, cudaStream_t st)
{
    if (b == 0 || n == 0) return cudaSuccess;
    if (off) kge_radius_kernel<true><<<(unsigned)b, RN_THREADS, 0, st>>>(chunk, ld, n, base, radius, cand_ids, cand_begin, cursor, off, nbr);
    else kge_radius_kernel<false><<<(unsigned)b, RN_THREADS, 0, st>>>(chunk, ld, n, base, radius, cand_ids, cand_begin, cursor, off, nbr);
    return cudaGetLastError();
}

__global__ void kge_radius_counts_kernel(const long long *__restrict__ cursor, long long b, long long *__restrict__ offsets)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) offsets[0] = 0;
    if (i < b) offsets[i + 1] = cursor[i];
}

cudaError_t launch_radius_counts(const long long *cursor, long long b, long long *offsets, cudaStream_t st)
{
    kge_radius_counts_kernel<<<(unsigned)((b + 256) / 256), 256, 0, st>>>(cursor, b, offsets);
    return cudaGetLastError();
}

}  // namespace kge
