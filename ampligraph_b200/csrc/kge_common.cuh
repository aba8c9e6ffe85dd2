// kge_common.cuh -- shared device helpers for libkge_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "../../include/kge_b200.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900 || !defined(__CUDA_ARCH_FEAT_SM90_ALL))
#error "libkge_b200 targets sm_90a (H100) only"
#endif

namespace kge {

// ---------------------------------------------------------------------------
// layout
// ---------------------------------------------------------------------------
struct Layout {
    int model;   // enum kge_scoring
    int k;       // user k
    int halves;  // 1 (TransE/DistMult) or 2 (ComplEx/HolE/RotatE)
    int kp;      // round_up(k, 4): floats per padded half
    int ld;      // halves * kp: row stride in floats
    int K;       // internal_k = halves * k
};

__host__ __device__ inline int model_halves(int model) { return (model == KGE_TRANSE || model == KGE_DISTMULT) ? 1 : 2; }

// ---------------------------------------------------------------------------
// warp helpers
// ---------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// ---------------------------------------------------------------------------
// fp32 pairs: two values in a 64-bit register pair.  Hopper has no packed fp32 instruction, so a pair operation is two
// IEEE fp32 operations (FFMA / FMUL / FADD, round to nearest), one per half; pk2 / upk2 are register renames.
// ---------------------------------------------------------------------------
typedef unsigned long long f32x2_t;
__device__ __forceinline__ f32x2_t pk2(float lo, float hi)
{
    f32x2_t r;
    asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
    return r;
}
__device__ __forceinline__ void upk2(f32x2_t v, float &lo, float &hi) { asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v)); }
__device__ __forceinline__ f32x2_t fma2(f32x2_t a, f32x2_t b, f32x2_t c)
{
    float a0, a1, b0, b1, c0, c1;
    upk2(a, a0, a1); upk2(b, b0, b1); upk2(c, c0, c1);
    return pk2(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
__device__ __forceinline__ f32x2_t mul2(f32x2_t a, f32x2_t b)
{
    float a0, a1, b0, b1;
    upk2(a, a0, a1); upk2(b, b0, b1);
    return pk2(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
__device__ __forceinline__ f32x2_t add2(f32x2_t a, f32x2_t b)
{
    float a0, a1, b0, b1;
    upk2(a, a0, a1); upk2(b, b0, b1);
    return pk2(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}
__device__ __forceinline__ f32x2_t sub2(f32x2_t a, f32x2_t b)
{
    float a0, a1, b0, b1;
    upk2(a, a0, a1); upk2(b, b0, b1);
    return pk2(__fsub_rn(a0, b0), __fsub_rn(a1, b1));
}

// ---------------------------------------------------------------------------
// PTX: mbarrier + 1-D bulk async copy (TMA engine, no tensor map) + bulk reduce
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init()
{
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem()
{
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE;\n"
        "bra WAIT_LOOP;\n"
        "DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
// global -> shared::cta, completion signalled on an mbarrier (complete_tx::bytes)
__device__ __forceinline__ void bulk_load(void *smem_dst, const void *gmem_src, uint32_t bytes, uint64_t *bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// shared::cta -> global with element-wise fp32 atomic add performed by the copy engine
__device__ __forceinline__ void bulk_reduce_add_f32(void *gmem_dst, const void *smem_src, uint32_t bytes)
{
    asm volatile("cp.reduce.async.bulk.global.shared::cta.bulk_group.add.f32 [%0], [%1], %2;" ::"l"(gmem_dst),
                 "r"(smem_u32(smem_src)), "r"(bytes)
                 : "memory");
}
// shared::cta -> global plain bulk store (copy engine)
__device__ __forceinline__ void bulk_store(void *gmem_dst, const void *smem_src, uint32_t bytes)
{
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gmem_dst), "r"(smem_u32(smem_src)),
                 "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ---------------------------------------------------------------------------
// PTX: per-thread async copies global -> shared (cp.async).  With valid false nothing is read and the destination is
// zero-filled.  The 16-byte copy bypasses L1 (.cg), the 4-byte one goes through it (.ca).
// ---------------------------------------------------------------------------
__device__ __forceinline__ void cp_async16(void *smem_dst, const void *gmem_src, bool valid)
{
    unsigned sz = valid ? 16u : 0u;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(sz)
                 : "memory");
}
__device__ __forceinline__ void cp_async4(void *smem_dst, const void *gmem_src, bool valid)
{
    unsigned sz = valid ? 4u : 0u;
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(sz)
                 : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
// wait until at most N of this thread's committed groups are still in flight
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// ---------------------------------------------------------------------------
// Philox4x32-10 (counter-based; the in-kernel replacement for TF's stateful
// tf.random.uniform draws at CorruptionGenerationLayerTrain.py:55-74)
// ---------------------------------------------------------------------------
struct u32x4 {
    uint32_t x, y, z, w;
};
__host__ __device__ inline u32x4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
                                               uint32_t k1)
{
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        uint64_t p0 = (uint64_t)M0 * c0, p1 = (uint64_t)M1 * c2;
        uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0;
        uint32_t hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
        uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += W0; k1 += W1;
    }
    return u32x4{c0, c1, c2, c3};
}
// one corruption draw for tile-order row r = j*B + i of training step `step`:
// keep_subj in {0,1} (uniform), replacement id uniform in [0, n_ent)
__host__ __device__ inline void draw_corruption(uint64_t seed, uint64_t step, uint64_t r, uint32_t n_ent,
                                                int *keep_subj, int *repl)
{
    u32x4 v = philox4x32_10((uint32_t)r, (uint32_t)(r >> 32), (uint32_t)step, (uint32_t)(step >> 32),
                            (uint32_t)seed, (uint32_t)(seed >> 32));
    *keep_subj = (int)(v.x & 1u);
    *repl = (int)(((uint64_t)v.y * (uint64_t)n_ent) >> 32);
}

// (key, val) is one of the n lexsorted pairs (keys[], vals[]): a lower-bound binary search over the pairs.  The filter
// of the negative samplers (kge_negatives.cu, kge_nscaching.cu): keys p * n_ent + kept entity, values the replaced one.
__device__ __forceinline__ bool known_pair(const long long *__restrict__ keys, const int32_t *__restrict__ vals, long long n,
                                           long long key, int val)
{
    long long lo = 0, hi = n;
    while (lo < hi) {
        const long long mid = (lo + hi) >> 1;
        const long long k = keys[mid];
        if (k < key || (k == key && vals[mid] < val)) lo = mid + 1;
        else hi = mid;
    }
    return lo < n && keys[lo] == key && vals[lo] == val;
}

// ---------------------------------------------------------------------------
// canonical arithmetic shared with the ranking oracle (oracle/kge_oracle.c states
// the same operation sequence independently): explicit _rn intrinsics so that
// nvcc never contracts or reassociates.
// ---------------------------------------------------------------------------
__device__ __forceinline__ double kge_poly_sin(double r)
{
    double r2 = __dmul_rn(r, r);
    double p = 2.81145725434552075980e-15;
    p = __fma_rn(p, r2, -7.64716373181981647590e-13);
    p = __fma_rn(p, r2, 1.60590438368216145994e-10);
    p = __fma_rn(p, r2, -2.50521083854417187751e-08);
    p = __fma_rn(p, r2, 2.75573192239858906526e-06);
    p = __fma_rn(p, r2, -1.98412698412698412698e-04);
    p = __fma_rn(p, r2, 8.33333333333333333333e-03);
    p = __fma_rn(p, r2, -1.66666666666666666667e-01);
    return __fma_rn(__dmul_rn(r, r2), p, r);
}
__device__ __forceinline__ double kge_poly_cos(double r)
{
    double r2 = __dmul_rn(r, r);
    double p = 4.77947733238738529744e-14;
    p = __fma_rn(p, r2, -1.14707455977297247139e-11);
    p = __fma_rn(p, r2, 2.08767569878680989792e-09);
    p = __fma_rn(p, r2, -2.75573192239858906526e-07);
    p = __fma_rn(p, r2, 2.48015873015873015873e-05);
    p = __fma_rn(p, r2, -1.38888888888888888889e-03);
    p = __fma_rn(p, r2, 4.16666666666666666667e-02);
    p = __fma_rn(p, r2, -5.00000000000000000000e-01);
    return __fma_rn(r2, p, 1.0);
}
// deterministic fp32 sin/cos (RotatE.py:97-98): fp64 Cody-Waite + Taylor, one rounding
__device__ __forceinline__ void kge_sincosf(float xf, float *s_out, float *c_out)
{
    double x = (double)xf;
    double n = rint(__dmul_rn(x, 6.36619772367581382433e-01));
    double r = __fma_rn(-n, 1.57079632679489655800e+00, x);
    r = __fma_rn(-n, 6.12323399573676603587e-17, r);
    double s = kge_poly_sin(r), c = kge_poly_cos(r);
    long long q = (long long)n & 3;
    double ss, cc;
    if (q == 0) { ss = s; cc = c; }
    else if (q == 1) { ss = c; cc = -s; }
    else if (q == 2) { ss = -s; cc = -c; }
    else { ss = -c; cc = s; }
    *s_out = (float)ss;
    *c_out = (float)cc;
}

__host__ inline float rotate_divisor(int K, long long n_rel)
{
    // RotatE.py:96-98: embedding_range = (6/(internal_k*max_rel_size))**0.5; theta/(range/pi)
    double range = sqrt(6.0 / ((double)K * (double)n_rel));
    return (float)(range / 3.14159265358979323846);
}
__host__ inline float hole_scale(int K) { return (float)(2.0 / ((double)K / 2.0)); }  // HolE.py:45

// AbstractScoringLayer.py:11,:201: int32(score * 1e3), truncation toward zero
__device__ __forceinline__ int quantise(float score) { return __float2int_rz(__fmul_rn(score, 1000.0f)); }

// ---------------------------------------------------------------------------
// host-side launch helpers
// ---------------------------------------------------------------------------
// Let kern use up to smem bytes of dynamic shared memory (a kernel gets 48 KB unless it is raised).  Occupancy queries
// for more than 48 KB need it too.
template <class Kernel>
static cudaError_t allow_dynamic_smem(Kernel kern, size_t smem)
{
    return cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
}

// Raise kern's shared-memory limit to smem bytes, launch, and return the launch's status
template <class Kernel, class... Args>
static cudaError_t launch_with_smem(Kernel kern, dim3 grid, int threads, size_t smem, cudaStream_t st, Args... args)
{
    cudaError_t e = allow_dynamic_smem(kern, smem);
    if (e != cudaSuccess) return e;
    kern<<<grid, threads, smem, st>>>(args...);
    return cudaGetLastError();
}

// Returns launch(std::integral_constant<int, V>) for the V of VS equal to v, the template arguments a launcher's kernel
// is instantiated for, or cudaErrorInvalidValue when v is none of them.
template <int... VS, class Launch>
static cudaError_t dispatch_value(int v, Launch &&launch)
{
    cudaError_t e = cudaErrorInvalidValue;
    (void)((v == VS && ((e = launch(std::integral_constant<int, VS>{})), true)) || ...);
    return e;
}

}  // namespace kge
