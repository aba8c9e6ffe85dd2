// kge_topk.cu -- exact top-k selection over candidate scores (sm_90a).
//
// Replaces the host side of discovery.query_topn (discovery.py:1143-1168): the reference scores every completed triple
// with model.predict and sorts all of them with np.argsort.  Here the candidate table is scored chunk by chunk by the
// ranking kernels (kge_rank.cu, canonical FP32 chain) into an L2-resident [b, C] buffer, and this file keeps a running
// top-k per query that each chunk is merged into, so no [b, n_cand] matrix is ever materialised.
//
// Ordering contract (the same in the host restatement of the tests and in DESIGN.md 3.6): score descending; equal
// scores by candidate position ascending, equality being float equality (-0 == +0); every NaN equal to every other NaN
// and above +inf.  One 64-bit key per (score, position) encodes it -- high word: the order-preserving uint32 image of
// the score with NaN canonicalised to 0x7fc00000 and -0 to +0, low word: 0xffffffff - position -- so "larger key first"
// is the whole rule, and keys of different candidates never compare equal.  Every key is > 0 (the smallest high word,
// that of -inf, is 0x007fffff), so 0 serves as "no threshold" and as the padding of the sort.
#include <math.h>

#include "kge_internal.h"

namespace kge {

constexpr int TK_THREADS = 512, TK_TILE = 4096, TK_PER = TK_TILE / TK_THREADS;

__device__ __forceinline__ unsigned long long topk_key(float s, long long pos)
{
    unsigned u = __float_as_uint(s);
    if ((u & 0x7fffffffu) > 0x7f800000u) u = 0x7fc00000u;  // NaN
    if (u == 0x80000000u) u = 0u;                          // -0
    const unsigned hi = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    return ((unsigned long long)hi << 32) | (0xffffffffu - (unsigned)pos);
}
__device__ __forceinline__ long long topk_pos(unsigned long long key) { return (long long)(0xffffffffu - (unsigned)key); }

// descending bitonic sort of s[0, n2), n2 a power of two, by the whole CTA; ends with a barrier
__device__ __forceinline__ void bitonic_desc(unsigned long long *s, int n2, int t)
{
    for (int k2 = 2; k2 <= n2; k2 <<= 1)
        for (int j = k2 >> 1; j > 0; j >>= 1) {
            for (int i = t; i < n2; i += TK_THREADS) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const unsigned long long a = s[i], b = s[ixj];
                    if (((i & k2) == 0) ? (a < b) : (a > b)) { s[i] = b; s[ixj] = a; }
                }
            }
            __syncthreads();
        }
}

// One CTA per query.  The query's running list -- at most k keys, descending, and the raw score of each (the key has
// lost the sign of zero and the NaN payload) -- lives in the workspace, double-buffered; state[q] = {entries, buffer}.
// The chunk is processed in tiles of TK_TILE columns:
//   1. tau = the k-th key of the list (0 while the list is not full);
//   2. if the query has filter entries, those inside the tile are marked in a shared bitmap; their keys become 0;
//   3. tau may be raised further (see below); keys > tau are compacted into shared memory (unordered);
//   4. the survivors are bitonic-sorted (descending, zero padded to a power of two);
//   5. the list and the survivors are merged into the other buffer, truncated to k: every element's output index is its
//      own index plus its co-rank in the other sequence (a binary search), which needs no partitioning pass.
// Once the list is full, tau is high and almost every tile ends after step 3: the kernel then reads the chunk once.
__global__ void __launch_bounds__(TK_THREADS) kge_topk_select_kernel(const TopkSelectParams p)
{
    __shared__ unsigned long long sk[TK_TILE];
    __shared__ unsigned bits[TK_TILE / 32];
    __shared__ int s_ns;
    const long long q = blockIdx.x;
    const int t = threadIdx.x, lane = t & 31;
    const size_t kk = (size_t)p.k, bk = (size_t)p.b * kk;
    const float *row = p.scores + (size_t)q * p.ld;
    const long long f0 = p.filt_off ? p.filt_off[q] : 0, f1 = p.filt_off ? p.filt_off[q + 1] : 0;
    const int2 st = p.state[q];
    int n = st.x, cur = st.y;  // CTA-uniform
    for (long long t0 = 0; t0 < p.n; t0 += TK_TILE) {
        const int tn = (int)(p.n - t0 < TK_TILE ? p.n - t0 : TK_TILE);
        const long long lo = p.base + t0;  // candidate position of the tile's first column
        const unsigned long long *ak = p.keys + cur * bk + q * kk;
        __syncthreads();  // the previous tile is done with sk, bits, s_ns, and its merge is visible
        unsigned long long tau = n == p.k ? ak[p.k - 1] : 0ull;
        if (t == 0) s_ns = 0;
        if (f1 > f0) {
            for (int i = t; i < TK_TILE / 32; i += TK_THREADS) bits[i] = 0u;
            __syncthreads();
            for (long long f = f0 + t; f < f1; f += TK_THREADS) {
                const long long c = (long long)p.filt_idx[f] - p.filt_shift - lo;
                if (c >= 0 && c < tn) atomicOr(&bits[c >> 5], 1u << (c & 31));
            }
            __syncthreads();
        }
        // key of column e * TK_THREADS + t; 0 past the tile and for filtered candidates.  Computed twice (maximum, then
        // compaction; the second read hits L1) rather than held: the held keys cost 16 registers and spilled.
        auto key_of = [&](int e) -> unsigned long long {
            const int c = e * TK_THREADS + t;
            const bool ok = c < tn && !(f1 > f0 && ((bits[c >> 5] >> (c & 31)) & 1u));
            return ok ? topk_key(row[t0 + c], lo + c) : 0ull;
        };
        unsigned long long mx = 0ull;
#pragma unroll
        for (int e = 0; e < TK_PER; ++e) {
            const unsigned long long v = key_of(e);
            mx = v > mx ? v : mx;
        }
        // While the list is short (the first tile of a query) every key passes tau, and sorting the whole tile to keep k
        // of it costs tens of microseconds of shared-memory traffic.  When at least k threads hold an eligible key above
        // tau, the k-th largest of the thread maxima is a lower bound of the k-th key of list + tile (k distinct keys
        // reach it): sorting the TK_THREADS maxima raises tau to just below it, and about k keys survive.
        const int active = __syncthreads_count(mx > tau);  // also the barrier after the reset of s_ns
        if (p.k <= TK_THREADS && active >= p.k && active > TK_THREADS / 4) {
            sk[t] = mx > tau ? mx : 0ull;
            __syncthreads();
            bitonic_desc(sk, TK_THREADS, t);
            const unsigned long long kth = sk[p.k - 1];
            __syncthreads();  // sk is reused by the compaction
            tau = kth - 1 > tau ? kth - 1 : tau;
        }
        // warp-aggregated compaction: one shared atomic per warp and column group (all lanes on one address would serialise)
#pragma unroll
        for (int e = 0; e < TK_PER; ++e) {
            const unsigned long long v = key_of(e);
            const bool keep = v > tau;
            const unsigned m = __ballot_sync(0xffffffffu, keep);
            if (m == 0u) continue;
            int at = 0;
            if (lane == 0) at = atomicAdd(&s_ns, __popc(m));
            at = __shfl_sync(0xffffffffu, at, 0);
            if (keep) sk[at + __popc(m & ((1u << lane) - 1u))] = v;
        }
        __syncthreads();
        const int nb = s_ns;
        if (nb == 0) continue;
        int n2 = 1;
        while (n2 < nb) n2 <<= 1;
        for (int i = nb + t; i < n2; i += TK_THREADS) sk[i] = 0ull;
        __syncthreads();
        bitonic_desc(sk, n2, t);
        const float *av = p.vals + cur * bk + q * kk;
        unsigned long long *ok = p.keys + (cur ^ 1) * bk + q * kk;
        float *ov = p.vals + (cur ^ 1) * bk + q * kk;
        for (int i = t; i < n; i += TK_THREADS) {
            const unsigned long long a = ak[i];
            int lo = 0, hi = nb;  // survivors greater than a
            while (lo < hi) { const int m = (lo + hi) >> 1; if (sk[m] > a) lo = m + 1; else hi = m; }
            const long long o = (long long)i + lo;
            if (o < p.k) { ok[o] = a; ov[o] = av[i]; }
        }
        for (int j = t; j < nb; j += TK_THREADS) {
            const unsigned long long v = sk[j];
            int lo = 0, hi = n;  // list entries greater than v
            while (lo < hi) { const int m = (lo + hi) >> 1; if (ak[m] > v) lo = m + 1; else hi = m; }
            const long long o = (long long)j + lo;
            if (o < p.k) { ok[o] = v; ov[o] = row[topk_pos(v) - p.base]; }
        }
        n = (long long)n + nb < p.k ? n + nb : p.k;
        cur ^= 1;
    }
    if (t == 0) p.state[q] = make_int2(n, cur);
}

// [b, k] outputs of the running lists: ids (cand_ids[pos], or cand_begin + pos; pos itself for kge_select_topk) and raw
// scores; rows with fewer than k eligible candidates are padded with id -1, score -inf.  NEG: every value is written
// negated, padding included (+inf) -- kge_knn stores -d to find the nearest points and reports d.
template <bool NEG>
__global__ void kge_topk_write_kernel(const int2 *__restrict__ state, const unsigned long long *__restrict__ keys,
                                      const float *__restrict__ vals, long long b, int k, const int32_t *__restrict__ cand_ids,
                                      long long cand_begin, int32_t *__restrict__ ids, float *__restrict__ out)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= b * k) return;
    const long long q = i / k;
    const int r = (int)(i - q * k);
    const int2 st = state[q];
    if (r < st.x) {
        const size_t src = (size_t)st.y * b * k + i;
        const long long pos = topk_pos(keys[src]);
        ids[i] = cand_ids ? cand_ids[pos] : (int32_t)(cand_begin + pos);
        out[i] = NEG ? -vals[src] : vals[src];
    } else {
        ids[i] = -1;
        out[i] = NEG ? INFINITY : -INFINITY;
    }
}

cudaError_t launch_topk_select(const TopkSelectParams &p, cudaStream_t st)
{
    if (p.b == 0 || p.n == 0) return cudaSuccess;
    kge_topk_select_kernel<<<(unsigned)p.b, TK_THREADS, 0, st>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_topk_write(const int2 *state, const unsigned long long *keys, const float *vals, long long b, int k,
                              const int32_t *cand_ids, long long cand_begin, int32_t *ids, float *out, cudaStream_t st,
                              bool negate)
{
    const long long n = b * k;
    if (n == 0) return cudaSuccess;
    auto kern = negate ? kge_topk_write_kernel<true> : kge_topk_write_kernel<false>;
    kern<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(state, keys, vals, b, k, cand_ids, cand_begin, ids, out);
    return cudaGetLastError();
}

}  // namespace kge
