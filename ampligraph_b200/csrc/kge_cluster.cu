// kge_cluster.cu -- DBSCAN over the rows of a point matrix (sm_90a): the device half of discovery.find_clusters.
//
// Replaces the host side of discovery.find_clusters (discovery.py:546-711) with its default algorithm, sklearn's
// DBSCAN: DBSCAN.fit runs a radius_neighbors self-join, keeps every neighbourhood in memory and labels the rows with
// sklearn.cluster._dbscan_inner.dbscan_inner.  Here the in-radius pairs are scored chunk by chunk by the ranking pair /
// tile kernel (the kge_radius_neighbors chunk loop, kge_api.cu) and consumed at once by the epilogues of this file, so
// no neighbourhood list is ever stored:
//   * union   -- every in-radius (query, candidate) pair of core rows joins the two ids in a union-find forest;
//   * min key -- for each query, the smallest key[c] over its in-radius candidates (border rows: the smallest root of
//                their core neighbours, i.e. the cluster dbscan_inner's depth-first search reaches first);
//   * flatten -- parent[x] = root(x).
//
// The forest, parent[n] (int32), is owned by the caller and starts as parent[x] = x.  Invariants:
//   (1) parent[x] <= x, and parent[x] < x for every non-root x, so every path strictly decreases and ends at the
//       smallest id of its tree.
//   (2) A hook is atomicCAS(&parent[hi], hi, lo) of the larger root hi to the smaller root lo.  A failed CAS means
//       another thread hooked hi first; the union retries from fresh finds.
//   (3) Every read of parent is ld.relaxed.gpu: it bypasses L1, which could otherwise hand a retrying thread the same
//       stale value forever.
//   (4) Path compression stores to parent[x] only after reading parent[x] != x.  A non-root never becomes a root
//       again, so the store cannot undo a hook (a store aimed at a root could land after another thread's CAS and
//       undo it).  The value stored is an ancestor read later along the path, so it is smaller and (1) holds.
// Termination: every store -- hook or compression -- lowers a parent value, and values are bounded below by 0, so
// finitely many stores happen; a find only follows strictly decreasing ids; a union retries only after another
// thread's hook succeeded.  Since the root of a tree is its smallest member whatever the order of the unions, the
// result is deterministic without ordered atomics.
#include <limits.h>

#include "kge_internal.h"

namespace kge {

constexpr int CL_THREADS = 512, CL_WARPS = CL_THREADS / 32;

__device__ __forceinline__ int parent_load(const int32_t *p)
{
    int v;
    asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

__device__ __forceinline__ void parent_store(int32_t *p, int v)
{
    asm volatile("st.relaxed.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// root of x with path halving: each visited non-root is pointed at its grandparent (invariant (4): x was read
// non-root before its store)
__device__ __forceinline__ int forest_find(int32_t *parent, int x)
{
    int p = parent_load(parent + x);
    while (p != x) {  // here p = a value read from parent[x], p != x
        const int g = parent_load(parent + p);
        if (g != p) parent_store(parent + x, g);
        x = p;
        p = g;
    }
    return x;
}

__device__ __forceinline__ void forest_union(int32_t *parent, int a, int b)
{
    for (;;) {
        a = forest_find(parent, a);
        b = forest_find(parent, b);
        if (a == b) return;
        const int hi = a > b ? a : b, lo = a > b ? b : a;
        if (atomicCAS(parent + hi, hi, lo) == hi) return;
        a = hi;  // hooked by another thread meanwhile: its new root is below hi
        b = lo;
    }
}

// One CTA per query row of a [b, ld] chunk of -d; columns [0, n) are candidate positions base + j.  The test is
// d <= radius, as in the radius epilogue of kge_knn.cu.
__global__ void __launch_bounds__(CL_THREADS) kge_radius_union_kernel(const float *__restrict__ chunk, long long ld,
                                                                      long long n, long long base, float radius,
                                                                      const int32_t *__restrict__ query_ids,
                                                                      const int32_t *__restrict__ cand_ids,
                                                                      long long cand_begin, int32_t *parent)
{
    const long long q = blockIdx.x;
    const float *row = chunk + (size_t)q * ld;
    const int a = query_ids[q];
    for (long long j = threadIdx.x; j < n; j += CL_THREADS) {
        if (!(-row[j] <= radius)) continue;
        const long long pos = base + j;
        const int c = cand_ids ? cand_ids[pos] : (int)(cand_begin + pos);
        if (c != a) forest_union(parent, a, c);
    }
}

cudaError_t launch_radius_union_chunk(const float *chunk, long long ld, long long n, long long base, long long b,
                                      float radius, const int32_t *query_ids, const int32_t *cand_ids,
                                      long long cand_begin, int32_t *parent, cudaStream_t st)
{
    if (b == 0 || n == 0) return cudaSuccess;
    kge_radius_union_kernel<<<(unsigned)b, CL_THREADS, 0, st>>>(chunk, ld, n, base, radius, query_ids, cand_ids,
                                                                 cand_begin, parent);
    return cudaGetLastError();
}

__global__ void kge_fill_i32_kernel(int32_t *__restrict__ x, long long n, int32_t v)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) x[i] = v;
}

cudaError_t launch_min_key_init(int32_t *out, long long b, cudaStream_t st)
{
    if (b == 0) return cudaSuccess;
    kge_fill_i32_kernel<<<(unsigned)((b + 255) / 256), 256, 0, st>>>(out, b, INT_MAX);
    return cudaGetLastError();
}

// out[q] = min(out[q], min key[c] over the chunk's in-radius candidates c); one CTA per query row.  A min is
// order-independent, so the result is deterministic.
__global__ void __launch_bounds__(CL_THREADS) kge_radius_min_key_kernel(const float *__restrict__ chunk, long long ld,
                                                                        long long n, long long base, float radius,
                                                                        const int32_t *__restrict__ cand_ids,
                                                                        long long cand_begin,
                                                                        const int32_t *__restrict__ key,
                                                                        int32_t *__restrict__ out)
{
    __shared__ int warp_min[CL_WARPS];
    const long long q = blockIdx.x;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    const float *row = chunk + (size_t)q * ld;
    int m = INT_MAX;
    for (long long j = t; j < n; j += CL_THREADS) {
        if (!(-row[j] <= radius)) continue;
        const long long pos = base + j;
        const int c = cand_ids ? cand_ids[pos] : (int)(cand_begin + pos);
        m = min(m, key[c]);
    }
    m = __reduce_min_sync(0xffffffffu, m);
    if (lane == 0) warp_min[warp] = m;
    __syncthreads();
    if (t == 0) {
#pragma unroll
        for (int w = 1; w < CL_WARPS; ++w) m = min(m, warp_min[w]);
        if (m < out[q]) out[q] = m;
    }
}

cudaError_t launch_radius_min_key_chunk(const float *chunk, long long ld, long long n, long long base, long long b,
                                        float radius, const int32_t *cand_ids, long long cand_begin,
                                        const int32_t *key, int32_t *out, cudaStream_t st)
{
    if (b == 0 || n == 0) return cudaSuccess;
    kge_radius_min_key_kernel<<<(unsigned)b, CL_THREADS, 0, st>>>(chunk, ld, n, base, radius, cand_ids, cand_begin,
                                                                   key, out);
    return cudaGetLastError();
}

// parent[x] = root(x), after the unions.  No compression on the way: a compression store could land after another
// thread's root store and put a non-root ancestor back.  Every store here writes a root, and a concurrent reader sees
// either the old ancestor or the root, both on the path.
__global__ void kge_forest_flatten_kernel(int32_t *parent, long long n)
{
    const long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= n) return;
    int r = (int)x, p = parent_load(parent + x);
    while (p != r) {
        r = p;
        p = parent_load(parent + r);
    }
    if (r != (int)x) parent_store(parent + x, r);
}

cudaError_t launch_forest_flatten(int32_t *parent, long long n, cudaStream_t st)
{
    if (n == 0) return cudaSuccess;
    kge_forest_flatten_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(parent, n);
    return cudaGetLastError();
}

}  // namespace kge
