// kge_graph.cu -- per-node wedge counts of an undirected simple graph (sm_90a): the device half of
// discovery.generate_candidates' graph strategies.
//
// Replaces nx.triangles, nx.clustering and nx.square_clustering (discovery.py:457-471 of the reference), which walk
// the graph node by node on the host.  With N(v) the neighbour set of v (self-loops removed), d(v) = |N(v)| and
// P(v, y) = |N(v) & N(y)| for y != v, the kernel writes for every node v
//   tri2[v] = sum_{u in N(v)} P(v, u)                                     (twice nx.triangles)
//   sq[v]   = sum_{y != v} P(v, y) (P(v, y) - 1) / 2                      (networkx's squares through v)
//   pot[v]  = (sum_{u in N(v)} d(u)) (d(v) - 1) - d(v)(d(v) - 1) - tri2[v] - sq[v]
// from which the three networkx statistics follow exactly on the host (DESIGN.md 3.9).
//
// Every P(v, y) is a count of wedges v - u - y (u in N(v), y in N(u), y != v).  One CTA at a time owns node v and a
// private counter array c[n_nodes] that is zero between nodes:
//   pass 1  c[y] += 1 for every wedge v - u - y                           -> c[y] = P(v, y)
//   pass 2  tri2 = sum_{u in N(v)} c[u]
//   pass 3  x = atomicExch(&c[y], 0) over the same wedges, sq += x (x - 1) / 2
// Pass 3 reads each y's final count exactly once (the first exchange takes it, later ones read 0) and leaves the
// array zero for the next node, so no memset runs between nodes.  The wedges of a node are enumerated flat: the
// neighbours are taken CTA-wide in chunks, an inclusive scan of their degrees maps wedge w to (u, position in N(u)),
// so a hub neighbour's list is spread over every thread instead of one warp.  Nodes come from an atomic work counter in
// the caller's order (heaviest first).  c lives in shared memory when it fits, else in the CTA's own slice of the
// workspace.  Every sum is int64 and every result an integer, so nothing depends on scheduling or on which path runs.
#include "kge_internal.h"

namespace kge {

constexpr int GR_THREADS = 512, GR_WARPS = GR_THREADS / 32;
constexpr int GR_GLOBAL_CTAS_PER_SM = 2;  // CTAs per SM of the workspace path (each owns n_nodes int32 counters)
constexpr size_t GR_HEADER = 256;         // workspace bytes before the counter slices: the work counter

struct GraphSmem {
    long long end[GR_THREADS];  // inclusive scan of the chunk's neighbour degrees
    long long beg[GR_THREADS];  // offsets[u] of the chunk's neighbours
    long long warp[GR_WARPS][3];
    long long item;
};

// inclusive scan of x over the CTA; ends with the CTA synchronised, returns the thread's inclusive prefix
__device__ __forceinline__ long long block_scan(long long x, GraphSmem &s)
{
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const long long y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) s.warp[warp][0] = x;
    __syncthreads();
    long long before = 0;
#pragma unroll
    for (int w = 0; w < GR_WARPS; ++w)
        if (w < warp) before += s.warp[w][0];
    __syncthreads();
    return x + before;
}

// op(y) for every wedge v - u - y with u in N(v) = nbr[b, e), y in N(u), y != v; returns sum_{u in N(v)} d(u) (the
// same value in every thread).  Ends with the CTA synchronised.
template <class Op>
__device__ __forceinline__ long long for_each_wedge(const long long *__restrict__ off, const int32_t *__restrict__ nbr,
                                                    int v, long long b, long long e, GraphSmem &s, Op op)
{
    const int t = threadIdx.x;
    long long wedges = 0;
    for (long long i0 = b; i0 < e; i0 += GR_THREADS) {
        const long long i = i0 + t;
        long long ub = 0, du = 0;
        if (i < e) {
            const int u = nbr[i];
            ub = off[u];
            du = off[u + 1] - ub;
        }
        const long long incl = block_scan(du, s);
        s.end[t] = incl;
        s.beg[t] = ub;
        __syncthreads();
        const int cnt = e - i0 < GR_THREADS ? (int)(e - i0) : GR_THREADS;
        const long long total = s.end[cnt - 1];
        int k = 0;  // w only grows, so the owning neighbour index only grows: search from the last one
        for (long long w = t; w < total; w += GR_THREADS) {
            int lo = k, hi = cnt - 1;  // smallest k with end[k] > w
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (s.end[mid] > w) hi = mid;
                else lo = mid + 1;
            }
            k = lo;
            const long long first = k ? s.end[k - 1] : 0;
            const int y = nbr[s.beg[k] + (w - first)];
            if (y != v) op(y);
        }
        wedges += total;
        __syncthreads();
    }
    return wedges;
}

__device__ __forceinline__ void block_sum3(long long a, long long b, long long c, GraphSmem &s, long long out[3])
{
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
        c += __shfl_xor_sync(0xffffffffu, c, o);
    }
    if (lane == 0) {
        s.warp[warp][0] = a;
        s.warp[warp][1] = b;
        s.warp[warp][2] = c;
    }
    __syncthreads();
    if (t == 0) {
        out[0] = out[1] = out[2] = 0;
#pragma unroll
        for (int w = 0; w < GR_WARPS; ++w) {
            out[0] += s.warp[w][0];
            out[1] += s.warp[w][1];
            out[2] += s.warp[w][2];
        }
    }
}

// kShared: c is the dynamic shared array; else c is this CTA's slice of `slices` (n int32 each).
template <bool kShared>
__global__ void __launch_bounds__(GR_THREADS) kge_graph_counts_kernel(const long long *__restrict__ off,
                                                                      const int32_t *__restrict__ nbr,
                                                                      const int32_t *__restrict__ order, long long n,
                                                                      unsigned long long *next, int32_t *slices,
                                                                      long long *__restrict__ tri2,
                                                                      long long *__restrict__ sq,
                                                                      long long *__restrict__ pot)
{
    extern __shared__ int32_t c_shared[];
    __shared__ GraphSmem s;
    const int t = threadIdx.x;
    int32_t *c = kShared ? c_shared : slices + (size_t)blockIdx.x * (size_t)n;
    for (long long i = t; i < n; i += GR_THREADS) c[i] = 0;
    for (;;) {
        if (t == 0) s.item = (long long)atomicAdd(next, 1ull);
        __syncthreads();  // also: c zeroed (first node), the previous node's sums read by thread 0
        const long long item = s.item;
        if (item >= n) return;
        const int v = order[item];
        const long long b = off[v], e = off[v + 1], dv = e - b;
        const long long deg_sum = for_each_wedge(off, nbr, v, b, e, s, [&](int y) { atomicAdd(c + y, 1); });
        long long t2 = 0;  // the workspace path reads through L2, where the atomics ran: L1 may hold a stale line
        for (long long i = b + t; i < e; i += GR_THREADS) t2 += kShared ? c[nbr[i]] : __ldcg(c + nbr[i]);
        __syncthreads();  // every c[u] read before pass 3 clears it
        long long s4 = 0;
        for_each_wedge(off, nbr, v, b, e, s, [&](int y) {
            const long long x = atomicExch(c + y, 0);
            s4 += x * (x - 1) / 2;
        });
        long long sum[3];
        block_sum3(t2, s4, 0, s, sum);
        if (t == 0) {
            tri2[v] = sum[0];
            sq[v] = sum[1];
            pot[v] = deg_sum * (dv - 1) - dv * (dv - 1) - sum[0] - sum[1];
        }
    }
}

// bytes of dynamic shared memory the shared-counter path needs for n nodes, or 0 if it does not fit on `dev`
static size_t shared_counter_bytes(long long n, int dev)
{
    int optin = 0;
    if (cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess) return 0;
    const size_t need = (size_t)n * sizeof(int32_t);
    return need + sizeof(GraphSmem) <= (size_t)optin ? need : 0;
}

static int global_ctas(int dev)
{
    int sms = 0;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
    return sms * GR_GLOBAL_CTAS_PER_SM;
}

long long graph_workspace_bytes(long long n)
{
    int dev = 0;
    if (n < 0 || cudaGetDevice(&dev) != cudaSuccess) return 0;
    if (n == 0 || shared_counter_bytes(n, dev) > 0) return (long long)GR_HEADER;
    const int ctas = global_ctas(dev);
    if (ctas == 0) return 0;
    return (long long)(GR_HEADER + (size_t)ctas * (size_t)n * sizeof(int32_t));
}

cudaError_t launch_graph_counts(const long long *off, const int32_t *nbr, const int32_t *order, long long n,
                                void *workspace, long long *tri2, long long *sq, long long *pot, cudaStream_t st)
{
    if (n == 0) return cudaSuccess;
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e != cudaSuccess) return e;
    unsigned long long *next = (unsigned long long *)workspace;
    e = cudaMemsetAsync(next, 0, sizeof(unsigned long long), st);
    if (e != cudaSuccess) return e;
    const size_t smem = shared_counter_bytes(n, dev);
    if (smem > 0) {
        e = allow_dynamic_smem(kge_graph_counts_kernel<true>, smem);
        if (e != cudaSuccess) return e;
        int per_sm = 0, sms = 0;
        e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kge_graph_counts_kernel<true>, GR_THREADS, smem);
        if (e != cudaSuccess) return e;
        e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        if (e != cudaSuccess) return e;
        long long grid = (long long)(per_sm > 0 ? per_sm : 1) * sms;
        if (grid > n) grid = n;
        kge_graph_counts_kernel<true><<<(unsigned)grid, GR_THREADS, smem, st>>>(off, nbr, order, n, next, nullptr, tri2,
                                                                                sq, pot);
    } else {
        // the slices must match graph_workspace_bytes, which sized them for global_ctas(dev) CTAs
        int32_t *slices = (int32_t *)((char *)workspace + GR_HEADER);
        long long grid = global_ctas(dev);
        if (grid > n) grid = n;
        kge_graph_counts_kernel<false><<<(unsigned)grid, GR_THREADS, 0, st>>>(off, nbr, order, n, next, slices, tri2,
                                                                               sq, pot);
    }
    return cudaGetLastError();
}

}  // namespace kge
