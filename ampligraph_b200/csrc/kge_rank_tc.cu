// kge_rank_tc.cu -- tensor-core FILTER pass of the all-entity ranking for the bilinear models (sm_90a: wgmma).
//
// For DistMult / ComplEx / HolE the corruption scores of a batch of queries are a contraction
// S[b, E] = Q[b, ld] . T[E, ld]^T (DistMult.py:51-99, ComplEx.py:65-151, HolE.py:47-89 compute it by broadcasting to
// [b, E, K]).  Ranks are counts of int32(score*1000) comparisons (AbstractScoringLayer.py:11,:201) and must be
// bit-identical to the canonical FP32 chain, which no tensor-core accumulation order reproduces.  But a rank only needs,
// per (query, candidate) pair, on which side of the positive's quantisation bin the candidate's score falls:
//
//   1. split      every fp32 operand x into two bf16 numbers, x ~ hi + lo (|x - hi - lo| <= 2^-16 |x|), laid out in HBM
//                 as ready-made wgmma operand tiles (8x8 "core matrices", K-major, no swizzle);
//   2. filter     (this kernel) approximate scores a = Qhi.Thi + Qhi.Tlo + Qlo.Thi on the tensor cores: wgmma.mma_async
//                 m64n256k16 (bf16 x bf16 -> fp32), accumulators in the registers of two consumer warpgroups, operand
//                 tiles staged by the copy engine (cp.async.bulk + mbarrier ring, one producer thread).  The epilogue
//                 compares a with the two edges U, L of the positive's bin: |a - s_canonical| <= delta is proven below, so a >= U + delta means
//                 "greater", L + delta <= a <= U - delta means "equal", a <= L - delta means "smaller";
//   3. refine     the few pairs inside a +-delta band around an edge are appended to a list and re-scored with the exact
//                 canonical chain (kge_rank_refine_kernel) -- same arithmetic as the FP32 kernel, same counters.
//   If the list overflows (it is sized for b*n_cand/16 pairs) the exact FP32 kernel redoes the whole call, gated on the
//   device-side counter: correctness never depends on the filter being selective.
//
// Error bound.  With u = 2^-8 (bf16 round-to-nearest): |x - hi| <= u|x|, |x - hi - lo| <= u^2 |x|.  The three computed
// products differ from q_d*e_d by the dropped terms lo*lo and the two residuals: <= 3 u^2 |q_d e_d| (+ O(u^3)); the
// bf16 x bf16 products themselves are exact in fp32.  The tensor core sums 3*ld products into an fp32 accumulator in an
// unspecified order; any order with fp32 roundings (truncation included, unit 2^-23) errs by <= 3 ld 2^-23 sum|q_d e_d|,
// and the canonical chain itself by <= ld 2^-24 sum|q_d e_d|.  With sum|q_d e_d| <= |q| |e| (Cauchy-Schwarz):
//     |a - s_canonical| <= (2^-14 + 4 ld 2^-23) |q|_2 |e|_2  =: eps_rel |q| |e|.
// tests/test_gpu_parity.py::test_tc_filter_error_bound measures the actual error (>= 10x smaller) and the bit-exact rank
// tests run both modes.
//
// Non-finite operands.  A NaN or inf in a query or candidate row makes its norm, and so delta, NaN or inf (a tile's norm
// is an atomicMax on the float bits, and NaN's bits are above every finite norm's); the filter takes an infinite delta
// as NaN, so every pair of that query or tile is undecided and goes to the refine (or, past the list's capacity, to the gated exact kernel).  Ranks stay exact;
// only the time such a broken table takes grows.  tests/test_gpu_rank_edges.py pins this.
#include <cuda_bf16.h>
#include <math.h>

#include "kge_rank_common.cuh"

namespace kge {

// ---------------------------------------------------------------------------------------------------------------------
// geometry
// ---------------------------------------------------------------------------------------------------------------------
constexpr int TC_MQ = 128;                         // queries per A tile    (two wgmma M = 64 halves, one per consumer warpgroup)
constexpr int TC_NC = 256;                         // candidates per B tile (wgmma N)
constexpr int TC_KB = 32;                          // columns per k-block (2 MMA k-steps of 16)
constexpr int TC_KC = TC_KB / 8;                   // 8-column chunks (core-matrix columns) per k-block
constexpr int TC_KSTEPS = TC_KB / 16;              // MMA k-steps per k-block
constexpr int TC_A_ELEMS = TC_MQ * TC_KB;          // bf16 elements of one part (hi or lo) of an A tile
constexpr int TC_B_ELEMS = TC_NC * TC_KB;
constexpr int TC_A_BYTES = 2 * TC_A_ELEMS * 2;     // hi + lo, contiguous in HBM and in shared memory: 16 KB
constexpr int TC_B_BYTES = 2 * TC_B_ELEMS * 2;     // 32 KB
constexpr int TC_STAGE_BYTES = TC_A_BYTES + TC_B_BYTES;  // 48 KB per pipeline stage
constexpr int TC_STAGES = 4;                       // operand ring depth: 192 KB of the 227 KB a block may use; the loop is bound by
                                                   // the latency of the bulk copies, so several smaller stages in flight beat
                                                   // fewer, larger ones
constexpr int TC_THREADS = 384;                    // warpgroup 0 producer, warpgroups 1-2 wgmma + epilogue

// ---------------------------------------------------------------------------------------------------------------------
// 1. split: fp32 rows -> blocked bf16 hi/lo operand tiles.
//    tile (rb, kb) of a matrix with RB rows per block: [hi: RB x TC_KB][lo: RB x TC_KB]; inside a part, element (r, c) lives
//    at ((r/8 * TC_KC + c/8) * 8 + r%8) * 8 + c%8: 8x8 core matrices of 128 contiguous bytes, TC_KC of them (one k-block)
//    per 8-row group -> the canonical K-major no-swizzle layout with LBO = 128 B (next k-chunk), SBO = TC_KC*128 B
//    (next 8-row group), so a whole tile is ONE contiguous bulk copy and needs no tensor map.
// ---------------------------------------------------------------------------------------------------------------------
// One WARP per row: lanes stride over the row's 8-column chunks (coalesced 32-byte reads), write the hi / lo core-matrix
// rows (16 bytes each) and accumulate the row's sum of squares on the way, so the norms the error bound needs cost no
// second pass.  Candidates (RB = 256): max |row| of each tile via atomicMax (positive floats order like their bit
// patterns).  Queries (RB = 128): the warp's lane 0 also writes the query's bin edges {U, L} in SCORE units (unscaled
// accumulator for HolE) and its error-bound factors.  qc >= n  <=>  trunc(x) >= n with x = fl(score*1000): x >= n for
// n >= 1, x > n-1 for n <= 0.
template <int RB>
__global__ void __launch_bounds__(256) kge_rank_split_kernel(const float *__restrict__ src, const int32_t *__restrict__ ids,
                                                             long long row_begin, long long n_rows, long long rows_pad,
                                                             int ld, int nkb, __nv_bfloat16 *__restrict__ out,
                                                             unsigned *__restrict__ tile_max, const int32_t *__restrict__ qpos,
                                                             float scale, float eps_rel, float4 *__restrict__ thr)
{
    const int lane = threadIdx.x & 31;
    const long long warp0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long n_warps = ((long long)gridDim.x * blockDim.x) >> 5;
    const int chunks = nkb * TC_KC;
    for (long long r = warp0; r < rows_pad; r += n_warps) {
        const bool live = r < n_rows;
        const float *row = live ? src + (size_t)(ids ? (long long)ids[r] : row_begin + r) * ld : nullptr;
        const long long rb = r / RB;
        const int rl = (int)(r - rb * RB);
        float ss = 0.f;
        for (int c = lane; c < chunks; c += 32) {
            const int kb = c / TC_KC, kc = c - kb * TC_KC, col0 = c * 8;
            float x[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            if (live) {
                if (col0 + 4 <= ld) { const float4 v = *reinterpret_cast<const float4 *>(row + col0); x[0] = v.x; x[1] = v.y; x[2] = v.z; x[3] = v.w; }
                if (col0 + 8 <= ld) { const float4 v = *reinterpret_cast<const float4 *>(row + col0 + 4); x[4] = v.x; x[5] = v.y; x[6] = v.z; x[7] = v.w; }
            }
            __align__(16) __nv_bfloat16 hi[8], lo[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                hi[e] = __float2bfloat16_rn(x[e]);
                lo[e] = __float2bfloat16_rn(x[e] - __bfloat162float(hi[e]));  // x - hi is exact in fp32
                ss = fmaf(x[e], x[e], ss);
            }
            const size_t tile = ((size_t)rb * nkb + kb) * (size_t)(2 * RB * TC_KB);
            const size_t off = (size_t)(((rl >> 3) * TC_KC + kc) * 8 + (rl & 7)) * 8;
            *reinterpret_cast<uint4 *>(out + tile + off) = *reinterpret_cast<const uint4 *>(hi);
            *reinterpret_cast<uint4 *>(out + tile + (size_t)RB * TC_KB + off) = *reinterpret_cast<const uint4 *>(lo);
        }
        ss = warp_sum(ss);
        if (lane != 0) continue;
        const float norm = __fmul_ru(__fsqrt_ru(ss), 1.00001f);  // rounded up: the sum's own rounding error is << 1e-5
        if (tile_max) {
            if (live) atomicMax(tile_max + rb, __float_as_uint(norm));
        } else if (!live) {
            thr[r] = make_float4(INFINITY, INFINITY, 0.f, 0.f);  // padding queries never count, never push
        } else {
            // in 64 bits: n + 1 must not wrap at INT_MAX.  quantise saturates, so nothing is greater than INT_MAX (U = +inf)
            // and nothing is smaller than INT_MIN (L = -inf)
            const long long n = qpos[r];
            const double edge_hi = (n + 1 >= 1) ? (double)(n + 1) : (double)n;  // T(n+1)
            const double edge_lo = (n >= 1) ? (double)n : (double)n - 1.0;      // T(n)
            const float U = n == INT_MAX ? INFINITY : (float)(edge_hi / 1000.0 / (double)scale);
            const float L = n == INT_MIN ? -INFINITY : (float)(edge_lo / 1000.0 / (double)scale);
            // slack: rounding of U, L themselves, of fl(scale*acc) and of fl(score*1000), each <= 2^-24 relative (64x margin);
            // from the finite edges only (an infinite one is never near a finite score)
            const float slack = fmaxf(n == INT_MAX ? 0.f : fabsf(U), n == INT_MIN ? 0.f : fabsf(L)) * 3.814697265625e-6f + 1e-37f;
            thr[r] = make_float4(U, L, __fmul_ru(eps_rel, norm), slack);
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// PTX wrappers: wgmma (warpgroup MMA, operands from shared memory, accumulators in registers)
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_arrive(uint64_t *bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait()
{
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// pins the accumulators after a wait: no use of them may move above it
__device__ __forceinline__ void acc_fence(float (&d)[128])
{
#pragma unroll
    for (int i = 0; i < 128; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D[64 x 256] (+)= A[64 x 16] . B[256 x 16]^T, bf16 x bf16 -> fp32, both operands K-major in shared memory; issued by the
// whole warpgroup.  Thread t of the warpgroup holds d[i] = D[16*(t/32) + (t%32)/4 + 8*((i/2)%2)][8*(i/4) + 2*(t%4) + i%2].
__device__ __forceinline__ void wgmma_m64n256k16_bf16(float (&d)[128], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate)
{
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
        "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
        "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
        "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
        "%128, %129, p, 1, 1, 0, 0;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
          "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
          "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
          "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
          "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
          "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
          "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
          "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
          "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate));
}

// shared-memory matrix descriptor (sm_90 wgmma): K-major, no swizzle (layout type 0), leading byte offset (next 8-column
// chunk along K) 128 B, stride byte offset (next 8-row group) TC_KC*128 B, base offset 0
__device__ __forceinline__ uint64_t wgmma_smem_desc(uint32_t smem_addr)
{
    return (uint64_t)((smem_addr >> 4) & 0x3fffu) | ((uint64_t)(128u >> 4) << 16) | ((uint64_t)((TC_KC * 128u) >> 4) << 32);
}

struct TcParams {
    const __nv_bfloat16 *a_split;  // [n_qb][nkb][hi|lo][128 x 32] query tiles
    const __nv_bfloat16 *b_split;  // [n_ct][nkb][hi|lo][256 x 32] candidate tiles
    const float4 *thr;             // [n_qb*128] {U, L, eps_rel*|q|, slack}
    const float *tile_norm;        // [n_ct] max |e| of the tile
    int32_t *cnt;                  // [b,3]
    int2 *pairs;                   // undecided (query, candidate position) pairs
    unsigned *pair_count;
    unsigned pair_cap;
    long long b, n_cand;
    int nkb, n_qb, n_ct, ctas_per_qb;
    float *probe_a, *probe_d;      // diagnostic outputs (PROBE instantiation only)
    float scale;
};

// ---------------------------------------------------------------------------------------------------------------------
// 2. the filter kernel.  CTA (qb, j): query block qb, candidate tiles j, j + ctas_per_qb, ...; one CTA per SM.
//    Warpgroup 0: one thread feeds a TC_STAGES-deep ring of {A tile + B tile} with bulk copies.  Warpgroups 1 and 2: query
//    rows 0-63 / 64-127 of the A tile against all 256 candidates of the B tile, 3 wgmma per k-step into 128 fp32 registers
//    per thread; one k-block stays in flight while the previous stage is released.  After the tile's last k-block each
//    thread compares its 128 accumulators (2 queries x 64 candidates) with the bin edges of its two queries.
// ---------------------------------------------------------------------------------------------------------------------
template <bool PROBE>
__global__ void __launch_bounds__(TC_THREADS, 1) kge_rank_tc_kernel(const TcParams p)
{
    extern __shared__ unsigned char tc_smem_raw[];
    unsigned char *smem = reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(tc_smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t *full = reinterpret_cast<uint64_t *>(smem + TC_STAGES * TC_STAGE_BYTES);  // [TC_STAGES] operands landed
    uint64_t *empty = full + TC_STAGES;                                        // [TC_STAGES] operands consumed
    const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
    const int qb = blockIdx.x % p.n_qb, first = blockIdx.x / p.n_qb;
    const int n_items = first < p.n_ct ? (p.n_ct - first + p.ctas_per_qb - 1) / p.ctas_per_qb : 0;

    if (threadIdx.x == 0) {
        for (int s = 0; s < TC_STAGES; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, 8); }  // empty: every consumer warp
        fence_mbar_init();
    }
    __syncthreads();

    if (wg == 0) {
        // ---------------- producer: one thread feeds the operand ring with bulk copies ----------------
        if (threadIdx.x == 0) {
            uint32_t it = 0;
            for (int i = 0; i < n_items; ++i) {
                const int ct = first + i * p.ctas_per_qb;
                for (int kb = 0; kb < p.nkb; ++kb, ++it) {
                    const int s = it % TC_STAGES;
                    mbar_wait(empty + s, ((it / TC_STAGES) & 1u) ^ 1u);
                    mbar_arrive_expect_tx(full + s, (uint32_t)TC_STAGE_BYTES);
                    unsigned char *st = smem + (size_t)s * TC_STAGE_BYTES;
                    bulk_load(st, p.a_split + ((size_t)qb * p.nkb + kb) * (size_t)(2 * TC_A_ELEMS), TC_A_BYTES, full + s);
                    bulk_load(st + TC_A_BYTES, p.b_split + ((size_t)ct * p.nkb + kb) * (size_t)(2 * TC_B_ELEMS), TC_B_BYTES, full + s);
                }
            }
        }
        return;
    }

    // ---------------- consumers: warpgroup cw owns query rows [64*cw, 64*cw + 64) of the tile ----------------
    const int cw = wg - 1;
    const int r0 = 64 * cw + 16 * warp + (lane >> 2);  // this thread's two queries: r0 and r0 + 8
    const long long q0 = (long long)qb * TC_MQ + r0, q1 = q0 + 8;
    const float4 thr0 = p.thr[q0], thr1 = p.thr[q1];
    const uint32_t a_row_off = (uint32_t)(64 * cw / 8) * (TC_KC * 128u);  // 8-row groups of the A tile before row 64*cw
    int gt0 = 0, ge0 = 0, gt1 = 0, ge1 = 0;
    uint32_t it = 0;
    float d[128];
    for (int i = 0; i < n_items; ++i) {
        const int ct = first + i * p.ctas_per_qb;
        int prev = -1;
        for (int kb = 0; kb < p.nkb; ++kb, ++it) {
            const int s = it % TC_STAGES;
            mbar_wait(full + s, (it / TC_STAGES) & 1u);
            const uint32_t a_hi = smem_u32(smem + (size_t)s * TC_STAGE_BYTES) + a_row_off, a_lo = a_hi + TC_A_ELEMS * 2;
            const uint32_t b_hi = smem_u32(smem + (size_t)s * TC_STAGE_BYTES) + TC_A_BYTES, b_lo = b_hi + TC_B_ELEMS * 2;
            wgmma_fence();
            // always TC_KSTEPS k-steps: the split kernel zero-fills every k-block past ld, and a trip count known at compile
            // time keeps the MMAs of one k-block in flight (a run-time bound makes ptxas serialise every wgmma)
#pragma unroll
            for (int ks = 0; ks < TC_KSTEPS; ++ks) {
                const uint32_t o = (uint32_t)ks * 256u;  // two 128-byte k-chunks per k-step of 16
                const uint64_t da_hi = wgmma_smem_desc(a_hi + o), da_lo = wgmma_smem_desc(a_lo + o);
                const uint64_t db_hi = wgmma_smem_desc(b_hi + o), db_lo = wgmma_smem_desc(b_lo + o);
                wgmma_m64n256k16_bf16(d, da_hi, db_hi, (kb | ks) != 0);
                wgmma_m64n256k16_bf16(d, da_hi, db_lo, 1u);
                wgmma_m64n256k16_bf16(d, da_lo, db_hi, 1u);
            }
            wgmma_commit();
            wgmma_wait<1>();  // the k-block before this one has completed: its stage may be overwritten
            if (prev >= 0 && lane == 0) mbar_arrive(empty + prev);
            prev = s;
        }
        wgmma_wait<0>();
        acc_fence(d);
        if (lane == 0) mbar_arrive(empty + prev);

        const long long c0 = (long long)ct * TC_NC;
        const int nvalid = (int)min((long long)TC_NC, p.n_cand - c0);
        const float tn = p.tile_norm[ct];
        // an infinite bound bounds nothing (an infinite score would compare >= it): NaN leaves every pair undecided
        const float dl0 = __fmaf_ru(__fmul_ru(thr0.z, tn), 1.0001f, thr0.w), delta0 = dl0 < INFINITY ? dl0 : NAN;
        const float dl1 = __fmaf_ru(__fmul_ru(thr1.z, tn), 1.0001f, thr1.w), delta1 = dl1 < INFINITY ? dl1 : NAN;
#pragma unroll
        for (int j = 0; j < 128; ++j) {
            const bool second = (j >> 1) & 1;
            const int col = 8 * (j >> 2) + 2 * (lane & 3) + (j & 1);
            const float a = d[j];
            const bool ok = col < nvalid;
            const float U = second ? thr1.x : thr0.x, L = second ? thr1.y : thr0.y, delta = second ? delta1 : delta0;
            const long long q = second ? q1 : q0;
            if (PROBE) {
                if (ok && q < p.b) {
                    p.probe_a[(size_t)q * p.n_cand + c0 + col] = a * p.scale;
                    p.probe_d[(size_t)q * p.n_cand + c0 + col] = delta * p.scale;
                }
                continue;
            }
            // written as !(>=) so that a NaN score and a NaN or infinite delta (a non-finite entry in the query, or in a row
            // of the tile: tile_norm is then NaN or inf) leave the pair undecided, for the exact refine to count
            const bool undecided = !(fminf(fabsf(a - U), fabsf(a - L)) >= delta);
            const int g = (ok && !undecided && a >= U) ? 1 : 0, e = (ok && !undecided && a >= L) ? 1 : 0;
            if (second) { gt1 += g; ge1 += e; } else { gt0 += g; ge0 += e; }
            if (ok && undecided) {
                const unsigned slot = atomicAdd(p.pair_count, 1u);
                if (slot < p.pair_cap) p.pairs[slot] = make_int2((int)q, (int)(c0 + col));
            }
        }
    }
    // the four threads of a quad share their two queries
#pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {
        gt0 += __shfl_xor_sync(0xffffffffu, gt0, o); ge0 += __shfl_xor_sync(0xffffffffu, ge0, o);
        gt1 += __shfl_xor_sync(0xffffffffu, gt1, o); ge1 += __shfl_xor_sync(0xffffffffu, ge1, o);
    }
    if ((lane & 3) == 0) {
        if (q0 < p.b) {
            if (gt0) atomicAdd(p.cnt + 3 * q0 + 0, gt0);
            if (ge0 - gt0) atomicAdd(p.cnt + 3 * q0 + 1, ge0 - gt0);
        }
        if (q1 < p.b) {
            if (gt1) atomicAdd(p.cnt + 3 * q1 + 0, gt1);
            if (ge1 - gt1) atomicAdd(p.cnt + 3 * q1 + 1, ge1 - gt1);
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// 3. refine: the exact canonical chain (same arithmetic as kge_rank_dot_kernel / the filter kernel of kge_rank.cu) for the
//    undecided pairs; one thread per pair.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void kge_rank_refine_kernel(const RankParams p, const int2 *__restrict__ pairs, const unsigned *__restrict__ pair_count,
                                       unsigned pair_cap, int32_t *__restrict__ cnt)
{
    extern __shared__ __align__(16) float pair_sm[];
    const unsigned n = *pair_count;
    if (n > pair_cap) {  // overflow: forget what the filter counted; the gated exact kernel (next launch) recounts everything
        for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < p.b; i += (long long)gridDim.x * blockDim.x) {
            cnt[3 * i] = 0;
            cnt[3 * i + 1] = 0;
        }
        return;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpc = blockDim.x >> 5;
    float *sm = pair_sm + (size_t)warp * 2 * p.L.ld;
    for (unsigned f = blockIdx.x * wpc + warp; f < n; f += gridDim.x * wpc) {  // one warp per undecided pair
        const int2 pr = pairs[f];
        const long long pos = pr.y;
        const long long id = p.cand_ids ? (long long)p.cand_ids[pos] : p.cand_begin + pos;
        const float sc = pair_score_warp<OP_DOT>(p.ent + (size_t)id * p.L.ld, p.qvec + (size_t)pr.x * p.L.ld, nullptr, p.L.ld, p.L.kp,
                                                 p.scale, sm, lane);
        if (lane == 0) {
            const int qc = quantise(sc), qp = p.qpos[pr.x];
            if (qp < qc) atomicAdd(cnt + 3 * pr.x + 0, 1);
            else if (qp == qc) atomicAdd(cnt + 3 * pr.x + 1, 1);
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------------
static size_t tc_align(size_t x) { return (x + 1023) & ~(size_t)1023; }

bool rank_tc_applicable(const Layout &L, int side, long long b, long long n_cand)
{
    (void)side;
    if (!(L.model == KGE_DISTMULT || L.model == KGE_COMPLEX || L.model == KGE_HOLE)) return false;
    // below this the FP32 kernel is already launch-bound; above, int positions / the per-SM query-block mapping must hold
    return b >= 1 && n_cand >= 512 && n_cand < (1ll << 31) && (b + TC_MQ - 1) / TC_MQ <= 128;
}

RankTcLayout rank_tc_layout(const Layout &L, long long b, long long n_cand, int pair_cap_override)
{
    RankTcLayout w;
    w.nkb = (L.ld + TC_KB - 1) / TC_KB;
    w.n_qb = (int)((b + TC_MQ - 1) / TC_MQ);
    w.n_ct = (int)((n_cand + TC_NC - 1) / TC_NC);
    long long cap = b * n_cand / 16;
    if (cap < (1ll << 20)) cap = 1ll << 20;
    if (cap > (1ll << 25)) cap = 1ll << 25;
    if (pair_cap_override > 0) cap = pair_cap_override;
    w.pair_cap = (unsigned)cap;
    size_t off = 0;
    w.off_a = off; off += tc_align((size_t)w.n_qb * w.nkb * TC_A_BYTES);
    w.off_b = off; off += tc_align((size_t)w.n_ct * w.nkb * TC_B_BYTES);
    w.off_thr = off; off += tc_align((size_t)w.n_qb * TC_MQ * sizeof(float4));
    w.off_count = off; off += 1024;                                       // pair counter, then the tile norms: one memset
    w.off_tnorm = off; off += tc_align((size_t)w.n_ct * sizeof(float));
    w.off_pairs = off; off += tc_align((size_t)w.pair_cap * sizeof(int2));
    w.bytes = off;
    return w;
}

cudaError_t launch_rank_count_tc(const RankParams &p, const RankTcLayout &w, void *ws, int32_t *cnt, int sm_count, cudaStream_t st,
                                 float *probe_a, float *probe_d)
{
    char *base = (char *)ws;
    __nv_bfloat16 *a_split = (__nv_bfloat16 *)(base + w.off_a), *b_split = (__nv_bfloat16 *)(base + w.off_b);
    float4 *thr = (float4 *)(base + w.off_thr);
    float *tnorm = (float *)(base + w.off_tnorm);
    unsigned *count = (unsigned *)(base + w.off_count);
    int2 *pairs = (int2 *)(base + w.off_pairs);
    const int ld = p.L.ld;
    cudaError_t e;
    if ((e = cudaMemsetAsync(count, 0, 1024 + (size_t)w.n_ct * sizeof(float), st)) != cudaSuccess) return e;
    // split (+ norms, + per-query thresholds): candidates in 256-row tiles, this side's query vectors in 128-row tiles
    const float eps_rel = (float)(ldexp(1.0, -14) + 4.0 * (double)ld * ldexp(1.0, -23));
    {
        const long long rows_pad = (long long)w.n_ct * TC_NC, want = (rows_pad + 7) / 8;
        kge_rank_split_kernel<TC_NC><<<(unsigned)(want < (long long)sm_count * 32 ? want : (long long)sm_count * 32), 256, 0, st>>>(
            p.ent, p.cand_ids, p.cand_begin, p.n_cand, rows_pad, ld, w.nkb, b_split, (unsigned *)tnorm, nullptr, 1.f, 0.f, nullptr);
    }
    {
        const long long rows_pad = (long long)w.n_qb * TC_MQ, want = (rows_pad + 7) / 8;
        kge_rank_split_kernel<TC_MQ><<<(unsigned)(want < (long long)sm_count * 32 ? want : (long long)sm_count * 32), 256, 0, st>>>(
            p.qvec, nullptr, 0, p.b, rows_pad, ld, w.nkb, a_split, nullptr, p.qpos, p.scale, eps_rel, thr);
    }
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    TcParams t;
    t.a_split = a_split; t.b_split = b_split; t.thr = thr; t.tile_norm = tnorm; t.cnt = cnt;
    t.pairs = pairs; t.pair_count = count; t.pair_cap = w.pair_cap;
    t.b = p.b; t.n_cand = p.n_cand; t.nkb = w.nkb; t.n_qb = w.n_qb; t.n_ct = w.n_ct;
    int per = sm_count / w.n_qb;
    if (per < 1) per = 1;
    if (per > w.n_ct) per = w.n_ct;
    t.ctas_per_qb = per;
    t.probe_a = probe_a; t.probe_d = probe_d; t.scale = p.scale;
    const size_t smem = (size_t)TC_STAGES * TC_STAGE_BYTES + 1024 /*alignment*/ + 128 /*barriers*/;
    const unsigned grid = (unsigned)(w.n_qb * per);
    if (probe_a) return launch_with_smem(kge_rank_tc_kernel<true>, grid, TC_THREADS, smem, st, t);
    if ((e = launch_with_smem(kge_rank_tc_kernel<false>, grid, TC_THREADS, smem, st, t)) != cudaSuccess) return e;
    const PairLaunch pl = pair_launch(ld, 2);
    if ((e = launch_with_smem(kge_rank_refine_kernel, sm_count * 2, pl.warps * 32, pl.smem, st, p, pairs, count, w.pair_cap, cnt)) !=
        cudaSuccess)
        return e;
    // overflow fallback: the exact FP32 kernel, every CTA of which returns at once unless the pair list overflowed
    RankParams g = p;
    g.gate = count;
    g.gate_cap = w.pair_cap;
    return launch_rank_count(g, cnt, st);
}

}  // namespace kge
