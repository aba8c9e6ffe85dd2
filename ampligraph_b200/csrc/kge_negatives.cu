// kge_negatives.cu -- the negative sampler of sampled training (kge_sample_negatives, DESIGN.md 3.18; sm_90a).
//
// Corruption r = j*B + i is the j-th corruption of positive i = (s, p, o), the tile order of the training kernels.  Its
// attempt a (0 <= a < max_attempts <= 256) uses the Philox4x32-10 block
//     v(a) = philox4x32_10((r_lo, r_hi | a << 24, step_lo, step_hi), (seed_lo, seed_hi)),
// which depends on (seed, step, r, a) only, and is draw_corruption's block at a = 0 (r < 2^56 keeps r_hi below 2^24).
//   side    from v(0) alone: without a threshold table keep = v.x & 1; with one, the subject is replaced (keep = 0) iff
//           v.x < thr[p]
//   entity  c = P[(v(a).y * |P|) >> 32], P the pool of (p, replaced side); all entities [0, n_ent) where there is no
//           pool or the pool row is empty (then c is draw_corruption's replacement at a = 0)
//   filter  while (s, p, c) (object replaced) or (c, p, o) (subject replaced) is a known triple and a + 1 < max_attempts,
//           draw c again from v(a + 1) (the side stays); a corruption still known after the last attempt is emitted and
//           counted in *misses.  Known = the (key, value) pair is in the side's lexsorted filter arrays, keys
//           p * n_ent + (kept entity), values the replaced entity (datasets.FilterIndex._obj / _sub).
// With no table, no pools and no filter the output is kge_generate_corruptions' stream.
#include "kge_internal.h"

namespace kge {

__device__ __forceinline__ u32x4 negative_block(const NegativeParams &p, unsigned long long r, unsigned a)
{
    return philox4x32_10((uint32_t)r, (uint32_t)(r >> 32) | (a << 24), (uint32_t)p.step, (uint32_t)(p.step >> 32),
                         (uint32_t)p.seed, (uint32_t)(p.seed >> 32));
}

__global__ void __launch_bounds__(256) kge_negatives_kernel(const NegativeParams p)
{
    const unsigned long long n = (unsigned long long)p.B * (unsigned long long)p.eta;
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    for (unsigned long long r = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += stride) {
        const long long i = (long long)(r % (unsigned long long)p.B);
        const int s = p.triples[3 * i], rel = p.triples[3 * i + 1], o = p.triples[3 * i + 2];
        const u32x4 v = negative_block(p, r, 0);
        const int keep = p.thr ? (v.x >= p.thr[rel] ? 1 : 0) : (int)(v.x & 1u);  // [keep]: 0 subject, 1 object replaced
        long long base = 0;
        unsigned long long len = p.n_ent;
        const int32_t *pool = nullptr;
        if (p.pool_off[keep]) {
            const long long lo = p.pool_off[keep][rel], hi = p.pool_off[keep][rel + 1];
            if (hi > lo) { base = lo; len = (unsigned long long)(hi - lo); pool = p.pool_ids[keep]; }
        }
        auto pick = [&](uint32_t y) {
            const long long q = (long long)(((unsigned long long)y * len) >> 32);
            return pool ? pool[base + q] : (int)q;
        };
        int c = pick(v.y);
        if (p.filt_n[keep] > 0) {
            const long long key = (long long)rel * (long long)p.n_ent + (keep ? s : o);
            for (unsigned a = 1; known_pair(p.filt_keys[keep], p.filt_vals[keep], p.filt_n[keep], key, c); ++a) {
                if (a >= (unsigned)p.max_attempts) {
                    if (p.misses) atomicAdd(p.misses, 1ull);
                    break;
                }
                c = pick(negative_block(p, r, a).y);
            }
        }
        p.neg_ent[r] = c;
        p.neg_keep[r] = (uint8_t)keep;
    }
}

cudaError_t launch_negatives(const NegativeParams &p, int sm_count, cudaStream_t st)
{
    const long long n = p.B * (long long)p.eta;
    if (n == 0) return cudaSuccess;
    const long long want = (n + 255) / 256, cap = 16ll * sm_count;
    kge_negatives_kernel<<<(unsigned)(want < cap ? want : cap), 256, 0, st>>>(p);
    return cudaGetLastError();
}

}  // namespace kge
