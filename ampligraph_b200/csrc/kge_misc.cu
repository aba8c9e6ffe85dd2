// kge_misc.cu -- predict-path scoring, layout packing, Glorot initialisation (sm_90a).
#include <math.h>

#include "kge_internal.h"

namespace kge {

// --------------------------------------------------------------------------
// predict_step (ScoringBasedEmbeddingModel.py:1694-1699): one warp per triple,
// rows read straight from HBM with coalesced 4-byte lanes (k values per half),
// warp-shuffle reduction.  Not the hot path; each score's error bound: tests/exact_oracle.py PredictBound.
// --------------------------------------------------------------------------
template <int MODEL>
__global__ void kge_score_kernel(const float *__restrict__ ent, const float *__restrict__ rel,
                                 const int32_t *__restrict__ triples, long long n, int k, int kp, int ld,
                                 float scale, float *__restrict__ out)
{
    const int lane = threadIdx.x & 31;
    const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long i = warp0; i < n; i += n_warps) {
        const float *s = ent + (size_t)triples[3 * i] * ld;
        const float *p = rel + (size_t)triples[3 * i + 1] * ld;
        const float *o = ent + (size_t)triples[3 * i + 2] * ld;
        float acc = 0.f;
        for (int d = lane; d < k; d += 32) {
            if (MODEL == KGE_TRANSE) {
                acc -= fabsf((s[d] + p[d]) - o[d]);
            } else if (MODEL == KGE_DISTMULT) {
                acc = fmaf(s[d] * p[d], o[d], acc);
            } else if (MODEL == KGE_COMPLEX || MODEL == KGE_HOLE) {
                float sr = s[d], si = s[kp + d], pr = p[d], pi = p[kp + d], orr = o[d], oi = o[kp + d];
                acc = fmaf(sr, fmaf(pi, oi, pr * orr), acc);
                acc = fmaf(si, fmaf(-pi, orr, pr * oi), acc);
            } else {  // RotatE: p is the rotation-table row [cos|sin]
                float sr = s[d], si = s[kp + d], c = p[d], sn = p[kp + d];
                float re = fmaf(-si, sn, sr * c) - o[d];
                float im = fmaf(si, c, sr * sn) - o[kp + d];
                acc -= sqrtf(fmaf(im, im, re * re));
            }
        }
        acc = warp_sum(acc);
        if (lane == 0) out[i] = scale * acc;
    }
}

cudaError_t launch_score_triples(const Layout &L, int, const float *ent, const float *rel_or_rot,
                                 const int32_t *triples, long long n, float scale, float *out, int sm_count,
                                 cudaStream_t st)
{
    if (n == 0) return cudaSuccess;
    const int threads = 256;
    long long want = (n + 7) / 8;
    int grid = (int)(want < (long long)sm_count * 8 ? want : (long long)sm_count * 8);
    return dispatch_value<KGE_TRANSE, KGE_DISTMULT, KGE_COMPLEX, KGE_HOLE, KGE_ROTATE>(L.model, [&](auto model) {
        kge_score_kernel<decltype(model)::value><<<grid, threads, 0, st>>>(ent, rel_or_rot, triples, n, L.k, L.kp, L.ld, scale, out);
        return cudaGetLastError();
    });
}

// --------------------------------------------------------------------------
// dense [rows, halves*k]  <->  padded [rows, halves*kp]
// --------------------------------------------------------------------------
__global__ void kge_pack_kernel(const float *__restrict__ src, float *__restrict__ dst, long long rows, int k,
                                int kp, int halves, bool unpack)
{
    const int ld = halves * kp, K = halves * k;
    long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= rows * ld) return;
    long long r = idx / ld;
    int c = (int)(idx - r * ld), h = c / kp, d = c - h * kp;
    if (unpack) {
        if (d < k) dst[r * K + h * k + d] = src[idx];
    } else {
        dst[idx] = (d < k) ? src[r * K + h * k + d] : 0.f;
    }
}

cudaError_t launch_pack(const Layout &L, const float *src, float *dst, long long rows, bool unpack, cudaStream_t st)
{
    long long n = rows * L.ld;
    if (n == 0) return cudaSuccess;
    kge_pack_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(src, dst, rows, L.k, L.kp, L.halves, unpack);
    return cudaGetLastError();
}

// --------------------------------------------------------------------------
// 'glorot_uniform' on shape [rows, internal_k] (EmbeddingLookupLayer.py:194-201):
// U(-l, l), l = sqrt(6/(fan_in+fan_out)) = sqrt(6/(rows+K)); pads stay 0.
// --------------------------------------------------------------------------
__global__ void kge_glorot_kernel(float *__restrict__ table, long long rows, int k, int kp, int halves,
                                  unsigned long long seed, float limit)
{
    const int ld = halves * kp;
    long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= rows * ld) return;
    long long r = idx / ld;
    int c = (int)(idx - r * ld), h = c / kp, d = c - h * kp;
    float v = 0.f;
    if (d < k) {
        unsigned long long e = (unsigned long long)r * (unsigned long long)(halves * k) + (unsigned long long)(h * k + d);
        u32x4 x = philox4x32_10((uint32_t)(e >> 2), (uint32_t)(e >> 34), 0x474c4f52u /*'GLOR'*/, 0u, (uint32_t)seed,
                                (uint32_t)(seed >> 32));
        uint32_t bits = (e & 3) == 0 ? x.x : (e & 3) == 1 ? x.y : (e & 3) == 2 ? x.z : x.w;
        float u = (float)(bits >> 8) * (1.0f / 16777216.0f);  // [0,1)
        v = fmaf(2.f * limit, u, -limit);
    }
    table[idx] = v;
}

// --------------------------------------------------------------------------
// The other initialisers tf.keras.initializers.get resolves (EmbeddingLookupLayer.py:105-129), reduced by the
// caller to four kinds.  One Philox4x32-10 block per element: x,y -> Box-Muller pair, z,w -> a second pair for
// the truncated normal's first resample; further resamples bump the counter's third word.
// --------------------------------------------------------------------------
__device__ __forceinline__ float u01(uint32_t bits) { return ((float)(bits >> 8) + 0.5f) * (1.0f / 16777216.0f); }  // (0,1)
__device__ __forceinline__ float box_muller(uint32_t a, uint32_t b)
{
    return sqrtf(-2.f * logf(u01(a))) * cospif(2.f * u01(b));
}

__global__ void kge_init_table_kernel(float *__restrict__ table, long long rows, int k, int kp, int halves, int kind,
                                      float a, float b, unsigned long long seed)
{
    const int ld = halves * kp;
    long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= rows * ld) return;
    long long r = idx / ld;
    int c = (int)(idx - r * ld), h = c / kp, d = c - h * kp;
    float v = 0.f;
    if (d < k) {
        const unsigned long long e = (unsigned long long)r * (unsigned long long)(halves * k) + (unsigned long long)(h * k + d);
        u32x4 x = philox4x32_10((uint32_t)e, (uint32_t)(e >> 32), 0x494e4954u /*'INIT'*/, 0u, (uint32_t)seed,
                                (uint32_t)(seed >> 32));
        if (kind == KGE_INIT_UNIFORM) {
            v = fmaf(b - a, (float)(x.x >> 8) * (1.0f / 16777216.0f), a);
        } else if (kind == KGE_INIT_NORMAL) {
            v = fmaf(b, box_muller(x.x, x.y), a);
        } else if (kind == KGE_INIT_TRUNCATED_NORMAL) {
            float n = box_muller(x.x, x.y);
            if (fabsf(n) > 2.f) n = box_muller(x.z, x.w);
            for (uint32_t t = 1; fabsf(n) > 2.f && t < 64u; ++t) {  // P(|n|>2) = 4.6 %: a handful of elements get here
                x = philox4x32_10((uint32_t)e, (uint32_t)(e >> 32), 0x494e4954u, t, (uint32_t)seed, (uint32_t)(seed >> 32));
                n = box_muller(x.x, x.y);
                if (fabsf(n) > 2.f) n = box_muller(x.z, x.w);
            }
            v = fmaf(b, fminf(fmaxf(n, -2.f), 2.f), a);
        } else {
            v = a;
        }
    }
    table[idx] = v;
}

cudaError_t launch_init_table(const Layout &L, float *table, long long rows, int kind, float a, float b,
                              unsigned long long seed, cudaStream_t st)
{
    long long n = rows * L.ld;
    if (n == 0) return cudaSuccess;
    kge_init_table_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(table, rows, L.k, L.kp, L.halves, kind, a, b, seed);
    return cudaGetLastError();
}

cudaError_t launch_glorot(const Layout &L, float *table, long long rows, unsigned long long seed, cudaStream_t st)
{
    long long n = rows * L.ld;
    if (n == 0) return cudaSuccess;
    float limit = (float)sqrt(6.0 / ((double)rows + (double)L.K));
    kge_glorot_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(table, rows, L.k, L.kp, L.halves, seed, limit);
    return cudaGetLastError();
}

}  // namespace kge
