// kge_optim.cu -- optimizer update of the embedding tables (sm_90a).
//
// Replaces OptimizerWrapper.minimize -> tf.keras.optimizers.legacy.*.apply_gradients
// (optimizers.py:136-168) and the regularisers attached to the tables
// (regularizers.py:14-37, EmbeddingLookupLayer.py:131-155; the per-element rules are in
// kge_optim_common.cuh), fused:
// one streaming pass reads {table, grad, slots}, writes {table, slots} and zeroes
// the gradient accumulator for the next step.  Semantics are the reference's
// DENSE ones: legacy Keras sums duplicate IndexedSlices rows first and Adam then
// decays m, v and moves EVERY row each step, touched or not (SURVEY.md 8a, A8).
// Bound: HBM, 8 fp32 streams per element for Adam (4 read + 4 written).
//
// Multi-GPU variants (replicated tables): kge_optim_sharded_kernel (one table, caller
// brackets it with barriers) and kge_optim_exchange_kernel (both tables, the cross-rank
// barriers are flag exchanges INSIDE the kernel: one launch per step).
#include <math.h>
#include <stdlib.h>

#include "kge_optim_common.cuh"

namespace kge {

template <int KIND, bool REG>
__global__ void __launch_bounds__(256) kge_optim_kernel(float4 *__restrict__ var, float4 *__restrict__ grad,
                                                        float4 *__restrict__ s0, float4 *__restrict__ s1,
                                                        long long n4, OptimParams o, double *reg_loss,
                                                        const OptimStep os)
{
    const bool S0 = uses_slot0(KIND, o.momentum), S1 = uses_slot1(KIND, o.momentum, o.centered);
    float racc = 0.f;
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        if constexpr (KIND == KGE_OPT_NADAM) {
            // row-decay mode (kge_optimizer_step_decay): a row that was not looked up only decays m and v; its table row
            // is not read or written, and its gradient row is already 0
            if (os.row_stamp && __ldg(os.row_stamp + i / os.ld4) != os.stamp) {
                float4 a4 = s0[i], b4 = s1[i];
                nadam_decay4(a4, b4, o);
                s0[i] = a4;
                s1[i] = b4;
                continue;
            }
        }
        float4 x4 = var[i], g4 = grad[i], a4 = z, b4 = z;
        if (S0) a4 = s0[i];
        if (S1) b4 = s1[i];
        var[i] = update4<KIND, REG>(x4, g4, a4, b4, o, os, o.reg, racc);
        if (S0) s0[i] = a4;
        if (S1) s1[i] = b4;
        grad[i] = z;
    }
    if (REG && reg_loss) flush_reg_loss(racc, reg_loss);
}

// --------------------------------------------------------------------------
// Data-parallel optimizer step FUSED with the gradient exchange over NVLink peer memory, ONE table.
// Tables are replicated, every rank holds a full gradient table produced by its own batch.
// Rank r owns the row shard [begin, end): it loads that shard of EVERY rank's gradient table
// (peer loads through NVSwitch), sums them in rank order (deterministic, identical on all
// ranks), applies the optimizer to its shard -- slots exist only for the shard -- and stores
// the updated parameters into EVERY rank's table (peer stores).  One kernel = reduce-scatter
// + sharded optimizer + all-gather.  The caller brackets it with two cross-rank barriers and
// zeroes its own gradient table afterwards (the row-sharded trainer uses it for the small,
// replicated relation table; the data-parallel trainer uses kge_optim_exchange_kernel).
// --------------------------------------------------------------------------
struct PeerPtrs {
    float4 *table[KGE_MAX_PEERS];
    const float4 *grad[KGE_MAX_PEERS];
};

template <int KIND, bool REG>
__global__ void __launch_bounds__(256) kge_optim_sharded_kernel(PeerPtrs pp, int world, int rank, float4 *__restrict__ s0,
                                                                float4 *__restrict__ s1, long long off4,
                                                                long long n4, OptimParams o, double *reg_loss,
                                                                const OptimStep os)
{
    const bool S0 = uses_slot0(KIND, o.momentum), S1 = uses_slot1(KIND, o.momentum, o.centered);
    float racc = 0.f;
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
        const long long gi = off4 + i;
        float4 gq[KGE_MAX_PEERS];
#pragma unroll
        for (int q = 0; q < KGE_MAX_PEERS; ++q)
            if (q < world) gq[q] = __ldcg(pp.grad[q] + gi);  // peer (or local) load, L2-coherent
        float4 g4 = z;
#pragma unroll
        for (int q = 0; q < KGE_MAX_PEERS; ++q)
            if (q < world) { g4.x += gq[q].x; g4.y += gq[q].y; g4.z += gq[q].z; g4.w += gq[q].w; }
        float4 x4 = pp.table[rank][gi], a4 = z, b4 = z;  // all replicas are identical; read the local one
        if (S0) a4 = s0[i];
        if (S1) b4 = s1[i];
        const float4 xn = update4<KIND, REG>(x4, g4, a4, b4, o, os, o.reg, racc);
#pragma unroll
        for (int q = 0; q < KGE_MAX_PEERS; ++q)
            if (q < world) __stcg(pp.table[q] + gi, xn);  // deliver the updated rows to every replica
        if (S0) s0[i] = a4;
        if (S1) s1[i] = b4;
    }
    if (REG && reg_loss) flush_reg_loss(racc, reg_loss);
}

cudaError_t launch_optimizer_sharded(const OptimParams &o, const OptimStep &os, int world, int rank, float *const *tables, float *const *grads,
                                     float *slot0, float *slot1, long long off_floats, long long n_floats,
                                     double *reg_loss, int sm_count, cudaStream_t st)
{
    long long n4 = n_floats / 4;
    if (n4 == 0) return cudaSuccess;
    PeerPtrs pp;
    for (int q = 0; q < KGE_MAX_PEERS; ++q) {
        pp.table[q] = q < world ? (float4 *)tables[q] : nullptr;
        pp.grad[q] = q < world ? (const float4 *)grads[q] : nullptr;
    }
    long long want = (n4 + 255) / 256;
    int grid = (int)(want < (long long)sm_count * 8 ? want : (long long)sm_count * 8);
    float4 *a = (float4 *)slot0, *b = (float4 *)slot1;
    const long long off4 = off_floats / 4;
    return dispatch_optimizer(o.kind, o.reg.p > 0, [&](auto kind, auto reg) {
        kge_optim_sharded_kernel<kind, reg><<<grid, 256, 0, st>>>(pp, world, rank, a, b, off4, n4, o, reg_loss, os);
        return cudaGetLastError();
    });
}

// --------------------------------------------------------------------------
// Cross-rank flag barrier over peer memory.  Every rank owns a pad of 2*world uint32 (slot s, writer
// q at pad[s*world + q]); a rank signals by storing a strictly increasing token into ITS entry of
// every rank's pad (st.release.sys through the peer mapping) and waits by polling its own pad
// (ld.acquire.sys, local memory).  Tokens only grow, so flags are never reset.
// --------------------------------------------------------------------------
__device__ __forceinline__ void st_release_sys(unsigned *p, unsigned v)
{
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned *p)
{
    unsigned v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
// token comparison that survives wrap-around of the 32-bit counter
__device__ __forceinline__ bool token_reached(unsigned seen, unsigned token) { return (int)(seen - token) >= 0; }

struct FlagPtrs {
    unsigned *pad[KGE_MAX_PEERS];
};
// thread q < world signals rank q; call from one warp
__device__ __forceinline__ void flags_signal(const FlagPtrs &f, int world, int rank, int slot, unsigned token, int lane)
{
    if (lane < world) st_release_sys(f.pad[lane] + slot * world + rank, token);
}
// thread q < world waits for rank q's signal in the local pad; call from one warp
__device__ __forceinline__ void flags_wait(const FlagPtrs &f, int world, int rank, int slot, unsigned token, int lane)
{
    if (lane < world) {
        const unsigned *p = f.pad[rank] + slot * world + lane;
        while (!token_reached(ld_acquire_sys(p), token)) __nanosleep(64);
    }
    __syncwarp();
}

__global__ void kge_peer_barrier_kernel(FlagPtrs f, int world, int rank, int slot, unsigned token)
{
    __threadfence_system();
    flags_signal(f, world, rank, slot, token, threadIdx.x);
    flags_wait(f, world, rank, slot, token, threadIdx.x);
}

cudaError_t launch_peer_barrier(int world, int rank, unsigned *const *flags, int slot, unsigned token, cudaStream_t st)
{
    FlagPtrs f;
    for (int q = 0; q < KGE_MAX_PEERS; ++q) f.pad[q] = q < world ? flags[q] : nullptr;
    kge_peer_barrier_kernel<<<1, 32, 0, st>>>(f, world, rank, slot, token);
    return cudaGetLastError();
}

// --------------------------------------------------------------------------
// The ONE-LAUNCH data-parallel step tail (kge_optimizer_step_exchange): both replicated tables as
// one contiguous [ent|rel] block.
//   phase 1  every CTA: warp 0 signals slot 0 (idempotent: all CTAs store the same token, so no CTA
//            depends on another CTA of this grid being scheduled) and waits until every rank has
//            entered the kernel -- i.e. finished its training kernel, by stream order: all gradient
//            blocks are complete.
//   phase 2  reduce-scatter + optimizer + all-gather over this rank's shard, 4 float4 per thread per
//            trip (4*world peer loads in flight per thread); the local NEXT-step gradient block is
//            zeroed on the way (gradient blocks are double-buffered, nobody memsets).
//   phase 3  each CTA fences its peer stores at system scope and counts itself done; the LAST CTA
//            signals slot 1 to every rank and waits for every rank's slot-1 token, which holds the
//            kernel open until all parameters destined for this rank have landed: the next kernel
//            on the stream may read the tables.
// --------------------------------------------------------------------------
// NVLS variant (MC = true): the gradient shard is reduced INSIDE the NVSwitch (multimem.ld_reduce on the multicast
// mapping of the gradient block: one load returns the sum over all ranks) and the updated rows are broadcast by the switch
// (multimem.st on the multicast mapping of the parameter block): per rank 1/N of a block crosses its links each way
// instead of (N-1)/N.  The switch fixes its own summation order, so results agree with the peer-load variant to fp32
// rounding, not bit for bit; replicas stay identical because every element still has exactly one writer.
__device__ __forceinline__ float4 multimem_ld_reduce_add(const float4 *mc)
{
    float4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                 : "l"(mc)
                 : "memory");
    return v;
}
__device__ __forceinline__ void multimem_st(float4 *mc, float4 v)
{
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
                 : "memory");
}

struct ExchangeArgs {
    float4 *table[KGE_MAX_PEERS];
    const float4 *grad[KGE_MAX_PEERS];
    float4 *table_mc;        // multicast mapping of the parameter block (MC instantiation) or nullptr
    const float4 *grad_mc;   // multicast mapping of this step's gradient block
    FlagPtrs flags;
    float4 *zero_grad;
    float4 *s0, *s1;
    long long total4, off4, n4, ent4;
    RegParams reg_ent, reg_rel;
    double *reg_loss;
    unsigned *done_counter;
    unsigned long long *trace;  // nullptr, or 8 x uint64 %globaltimer stamps of the phases (kge_set_exchange_trace)
    unsigned token;
    int world, rank, phases;
};
__device__ __forceinline__ unsigned long long globaltimer_ns()
{
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
// phase stamp by CTA 0 (or whoever is told to): one store, only when tracing
#define KGE_TRACE(slot, cond)                                                         \
    do {                                                                              \
        if (x.trace && (cond) && threadIdx.x == 0) x.trace[slot] = globaltimer_ns(); \
    } while (0)

template <int KIND, bool REG, int WORLD, bool MC>
__global__ void __launch_bounds__(256) kge_optim_exchange_kernel(const ExchangeArgs x, const OptimParams o,
                                                                    const OptimStep os)
{
    const bool S0 = uses_slot0(KIND, o.momentum), S1 = uses_slot1(KIND, o.momentum, o.centered);
    constexpr int U = WORLD <= 4 ? 4 : 2;  // float4s per thread per trip (U*WORLD peer loads in flight per thread)
    const int rank = x.rank;
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long nthreads = (long long)gridDim.x * blockDim.x;

    KGE_TRACE(0, blockIdx.x == 0);
    // phase 1a: announce this rank's arrival FIRST.  The release only has to cover the training kernel's gradient
    // scatters (complete at the kernel boundary); issued after the zeroing below it would also wait for those stores.
    if ((x.phases & 1) && threadIdx.x < 32) flags_signal(x.flags, WORLD, rank, 0, x.token, threadIdx.x);
    // zero the next step's local gradient block: independent of the peers, overlaps the barrier wait
    if (x.zero_grad)
        for (long long i = tid; i < x.total4; i += nthreads) __stcg(x.zero_grad + i, z);
    KGE_TRACE(1, blockIdx.x == 0);

    if (x.phases & 1) {  // phase 1b: every rank has entered the kernel
        if (threadIdx.x < 32) flags_wait(x.flags, WORLD, rank, 0, x.token, threadIdx.x);
        __syncthreads();
    }
    KGE_TRACE(2, blockIdx.x == 0);

    float racc = 0.f;
    // one element: optimizer on the summed gradient g4, new parameters delivered to every replica
    auto update_and_deliver = [&](long long i, float4 g4) {
        const long long gi = x.off4 + i;
        float4 x4 = x.table[rank][gi], a4 = z, b4 = z;
        if (S0) a4 = x.s0[i];
        if (S1) b4 = x.s1[i];
        // REG holds when either table has a regulariser; the other one (p = 0) takes the rule without it -- reg_grad
        // would form lam*0*powf(|x|, -1), NaN at x = 0, and add lam per element to the loss
        const RegParams &reg = gi < x.ent4 ? x.reg_ent : x.reg_rel;
        const float4 xn = (REG && reg.p > 0) ? update4<KIND, REG>(x4, g4, a4, b4, o, os, reg, racc)
                                             : update4<KIND, false>(x4, g4, a4, b4, o, os, reg, racc);
        if (MC) {
            multimem_st(x.table_mc + gi, xn);
        } else {
#pragma unroll
            for (int q = 0; q < WORLD; ++q) __stcg(x.table[q] + gi, xn);
        }
        if (S0) x.s0[i] = a4;
        if (S1) x.s1[i] = b4;
    };
    if constexpr (MC) {
        // NVLS: the reduce (multimem.ld_reduce: this GPU SENDS its share of every shard) and the broadcast (multimem.st:
        // this GPU RECEIVES every other shard) load opposite directions of the links, so they are software-pipelined:
        // the loads of trip t+1 are in flight while trip t is updated and broadcast (the grid is sized for a few trips).
        const long long stride = nthreads * U;
        float4 cur[U], nxt[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const long long i = tid + u * nthreads;
            if (i < x.n4) cur[u] = multimem_ld_reduce_add(x.grad_mc + x.off4 + i);
        }
        for (long long base = tid; base < x.n4; base += stride) {
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const long long i = base + stride + u * nthreads;
                if (i < x.n4) nxt[u] = multimem_ld_reduce_add(x.grad_mc + x.off4 + i);
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const long long i = base + u * nthreads;
                if (i < x.n4) update_and_deliver(i, cur[u]);
                cur[u] = nxt[u];
            }
        }
    } else {
        for (long long base = tid; base < x.n4; base += nthreads * U) {
            float4 gq[U][WORLD];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const long long i = base + u * nthreads;
                if (i < x.n4) {
#pragma unroll
                    for (int q = 0; q < WORLD; ++q) gq[u][q] = __ldcg(x.grad[q] + x.off4 + i);
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const long long i = base + u * nthreads;
                if (i >= x.n4) continue;
                float4 g4 = gq[u][0];
#pragma unroll
                for (int q = 1; q < WORLD; ++q) { g4.x += gq[u][q].x; g4.y += gq[u][q].y; g4.z += gq[u][q].z; g4.w += gq[u][q].w; }
                update_and_deliver(i, g4);
            }
        }
    }
    if (REG && x.reg_loss) flush_reg_loss(racc, x.reg_loss);

    KGE_TRACE(3, blockIdx.x == 0);
    if (x.phases & 2) {
        // Release pattern at CTA granularity: the CTA barrier orders every thread's peer stores before thread 0's
        // system-scope fence (fences are cumulative), which orders them before its done-count; the last CTA fences again
        // before it signals the peers.  One MEMBAR.SYS per CTA instead of one per thread.
        __syncthreads();
        __shared__ int last;
        if (threadIdx.x == 0) {
            __threadfence_system();
            last = (atomicAdd(x.done_counter, 1u) == gridDim.x - 1) ? 1 : 0;
        }
        __syncthreads();
        KGE_TRACE(4, blockIdx.x == 0);
        if (last && threadIdx.x < 32) {
            if (threadIdx.x == 0) *x.done_counter = 0u;  // self-reset for the next launch (stream-ordered)
            __threadfence_system();
            KGE_TRACE(5, true);
            flags_signal(x.flags, WORLD, rank, 1, x.token, threadIdx.x);
            flags_wait(x.flags, WORLD, rank, 1, x.token, threadIdx.x);
            KGE_TRACE(6, true);
        }
    }
}

// One instantiation of the exchange kernel, on a grid that is CO-RESIDENT: no CTA waits for another CTA of the grid, so a
// second wave would be correct -- but it starts only when first-wave CTAs retire, i.e. after their system-scope fence, and
// then runs its share of the exchange alone.  With the grid fixed at 4 CTAs per SM the 70-register variants (3 resident
// CTAs per SM: world 2) ran a quarter of the shard in such a second wave, and waiting for the last CTA took a large part of
// the kernel (measured before the H100 port).  The loops are grid-stride, so fewer CTAs only
// means more trips per thread.
template <int KIND, bool REG, int WORLD, bool MC>
static cudaError_t launch_exchange_variant(const ExchangeArgs &a, const OptimParams &o, const OptimStep &os, long long want,
                                           int sm_count, cudaStream_t st)
{
    auto kern = kge_optim_exchange_kernel<KIND, REG, WORLD, MC>;
    static int occ_cached = 0;  // per instantiation; the query is cheap but this is the per-step path
    if (occ_cached == 0) {
        int occ = 0;
        cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, 256, 0);
        if (e != cudaSuccess) return e;
        occ_cached = occ < 1 ? 1 : (occ > 4 ? 4 : occ);
    }
    const long long cap = (long long)sm_count * occ_cached;
    kern<<<(int)(want < cap ? want : cap), 256, 0, st>>>(a, o, os);
    return cudaGetLastError();
}

cudaError_t launch_optimizer_exchange(const OptimParams &o, const OptimStep &os, const ExchangeParams &xp, int sm_count, cudaStream_t st)
{
    ExchangeArgs a;
    for (int q = 0; q < KGE_MAX_PEERS; ++q) {
        a.table[q] = q < xp.world ? (float4 *)xp.table[q] : nullptr;
        a.grad[q] = q < xp.world ? (const float4 *)xp.grad[q] : nullptr;
        a.flags.pad[q] = q < xp.world ? xp.flags[q] : nullptr;
    }
    a.table_mc = (float4 *)xp.table_mc;
    a.grad_mc = (const float4 *)xp.grad_mc;
    const bool mc = xp.table_mc != nullptr && xp.grad_mc != nullptr;
    a.zero_grad = (float4 *)xp.zero_grad;
    a.s0 = (float4 *)xp.slot0;
    a.s1 = (float4 *)xp.slot1;
    a.total4 = xp.total4; a.off4 = xp.off4; a.n4 = xp.n4; a.ent4 = xp.ent4;
    a.reg_ent = xp.reg_ent; a.reg_rel = xp.reg_rel;
    a.reg_loss = xp.reg_loss;
    a.done_counter = xp.done_counter;
    a.trace = xp.trace;
    a.token = xp.token;
    a.world = xp.world; a.rank = xp.rank; a.phases = xp.phases;
    // no CTA ever waits for another CTA of this grid (phase 1 is per CTA, phase 3 is the last finisher alone), so the
    // grid need not be co-resident; a few CTAs per SM are enough to keep the NVLink loads in flight
    // grid: up to 4 CTAs per SM; the NVLS variant is software-pipelined, so it wants a few trips per thread rather than
    // every load of the shard in flight at once (KGE_B200_EXCHANGE_TRIPS, default 1 = one trip)
    int trips = 1;
    if (const char *e = getenv("KGE_B200_EXCHANGE_TRIPS")) trips = atoi(e) > 0 ? atoi(e) : 1;
    const int U = xp.world <= 4 ? 4 : 2;
    long long want = (a.n4 + 256LL * U * trips - 1) / (256LL * U * trips);
    const long long zero_want = (a.total4 / 8 + 255) / 256;  // the zeroing of the next gradient block wants enough threads too
    if (!mc || trips <= 1) want = want > zero_want ? want : zero_want;
    if (want < 1) want = 1;
    return dispatch_optimizer(o.kind, xp.reg_ent.p > 0 || xp.reg_rel.p > 0, [&](auto kind, auto reg) {
        auto variant = [&](auto world) {
            constexpr int K = decltype(kind)::value;
            constexpr bool R = decltype(reg)::value;
            return mc ? launch_exchange_variant<K, R, world, true>(a, o, os, want, sm_count, st)
                      : launch_exchange_variant<K, R, world, false>(a, o, os, want, sm_count, st);
        };
        return dispatch_value<1, 2, 3, 4, 5, 6, 7, 8>(xp.world, variant);
    });
}

// --------------------------------------------------------------------------
// LAZY optimizer (extension for tables whose dense update is unaffordable, e.g. cfg5: 10 M entities x
// k=1000 -> 80 GB table, 560 GB of dense-Adam traffic per step; SURVEY.md 8a A8).  Only rows stamped by
// this step's training kernel are read and updated: m, v of untouched rows do NOT decay and the rows do
// not move (the semantics of TensorFlow-Addons' LazyAdam), bias correction uses the global step.  This
// is NOT the reference's dense rule; it is opt-in ('lazy_adam' etc.).  A warp scans 32 row stamps with
// one coalesced read, ballots the touched ones and updates each touched row cooperatively.
// --------------------------------------------------------------------------
template <int KIND, bool REG>
__global__ void __launch_bounds__(256) kge_optim_lazy_kernel(float *__restrict__ var, float *__restrict__ grad,
                                                             float *__restrict__ s0, float *__restrict__ s1,
                                                             long long rows, int ld, const int *__restrict__ row_stamp,
                                                             int stamp, OptimParams o, double *reg_loss,
                                                             const OptimStep os)
{
    const bool S0 = uses_slot0(KIND, o.momentum), S1 = uses_slot1(KIND, o.momentum, o.centered);
    const int lane = threadIdx.x & 31;
    const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    float racc = 0.f;
    for (long long base = warp0 * 32; base < rows; base += n_warps * 32) {
        const long long r = base + lane;
        unsigned m = __ballot_sync(0xffffffffu, r < rows && row_stamp[r] == stamp);
        while (m) {
            const int b = __ffs(m) - 1;
            m &= m - 1;
            const size_t off = (size_t)(base + b) * ld;
            for (int c = lane * 4; c < ld; c += 128) {
                float4 x4 = *reinterpret_cast<float4 *>(var + off + c), g4 = *reinterpret_cast<float4 *>(grad + off + c);
                float4 a4 = z, b4 = z;
                if (S0) a4 = *reinterpret_cast<float4 *>(s0 + off + c);
                if (S1) b4 = *reinterpret_cast<float4 *>(s1 + off + c);
                *reinterpret_cast<float4 *>(var + off + c) = update4<KIND, REG>(x4, g4, a4, b4, o, os, o.reg, racc);
                if (S0) *reinterpret_cast<float4 *>(s0 + off + c) = a4;
                if (S1) *reinterpret_cast<float4 *>(s1 + off + c) = b4;
                *reinterpret_cast<float4 *>(grad + off + c) = z;
            }
        }
    }
    if (REG && reg_loss) {
        racc = warp_sum(racc);
        if (lane == 0 && racc != 0.f) atomicAdd(reg_loss, (double)racc);
    }
}

cudaError_t launch_optimizer_lazy(const OptimParams &o, const OptimStep &os, float *table, float *grad, float *slot0, float *slot1,
                                  long long rows, int ld, const int *row_stamp, int stamp, double *reg_loss,
                                  int sm_count, cudaStream_t st)
{
    if (rows == 0) return cudaSuccess;
    long long want = (rows + 255) / 256;  // 8 warps x 32 rows per block
    int grid = (int)(want < (long long)sm_count * 8 ? want : (long long)sm_count * 8);
    return dispatch_optimizer(o.kind, o.reg.p > 0, [&](auto kind, auto reg) {
        kge_optim_lazy_kernel<kind, reg><<<grid, 256, 0, st>>>(table, grad, slot0, slot1, rows, ld, row_stamp, stamp, o, reg_loss, os);
        return cudaGetLastError();
    });
}

cudaError_t launch_optimizer(const OptimParams &o, const OptimStep &os, float *table, float *grad, float *slot0, float *slot1,
                             long long n_floats, double *reg_loss, int sm_count, cudaStream_t st)
{
    long long n4 = n_floats / 4;  // ld is a multiple of 4
    if (n4 == 0) return cudaSuccess;
    long long want = (n4 + 255) / 256;
    int grid = (int)(want < (long long)sm_count * 8 ? want : (long long)sm_count * 8);
    float4 *v = (float4 *)table, *g = (float4 *)grad, *a = (float4 *)slot0, *b = (float4 *)slot1;
    return dispatch_optimizer(o.kind, o.reg.p > 0, [&](auto kind, auto reg) {
        kge_optim_kernel<kind, reg><<<grid, 256, 0, st>>>(v, g, a, b, n4, o, reg_loss, os);
        return cudaGetLastError();
    });
}

}  // namespace kge
