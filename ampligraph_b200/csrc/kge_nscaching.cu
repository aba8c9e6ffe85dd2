// kge_nscaching.cu -- NSCaching negative sampling (Zhang, Yao, Shao and Chen, ICDE 2019): per-query caches of
// high-scoring entities, refreshed by importance sampling and drawn from uniformly (kge_nscaching_step, DESIGN.md 3.20;
// sm_90a).
//
// Arrays indexed [side] are [0] for the subject-replaced caches, one row per distinct (p, o), and [1] for the
// object-replaced ones, one row per distinct (s, p) (= keep_subj, as in kge_negatives.cu).  Row `row` of a side holds
// count[row] <= N1 distinct entity ids in ids[row * N1 ..].  A step runs two kernels:
//   refresh  one CTA per (positive i, side) whose update flag is set (the first positive of the batch with that key).
//            Candidates c = 0, 1, ...: the row's count cached ids in stored order, then N2 draws e_j = (w * n_ent) >> 32,
//            w word j & 3 of philox4x32_10((row, (j >> 2) | side << 31, step_lo, step_hi), (seed_lo, seed_hi ^ NSC_KEY)).
//            A candidate equal to an earlier one, with a NaN score, or (filter) whose corrupted triple is known is
//            dropped.  Score: the canonical chain of kge_corruption_scores (kge_rank_common.cuh), one thread per
//            candidate.  Key = fl(score + G), G = -logf(-logf(u)), u = ((w' >> 9) + 0.5) 2^-23 (exact in fp32), w' word
//            c & 3 of the block with counter (row, (c >> 2) | 1 << 30 | side << 31, step_lo, step_hi).  The min(N1, valid)
//            valid candidates with the largest keys (ties: lower c) are kept -- Gumbel-top-k, a draw without replacement
//            with probability proportional to exp(score) -- and written back in ascending c.
//   draw     one thread per corruption r = j*B + i: v = the block of draw_corruption, side = v.x & 1, n = count of the
//            positive's row of that side; the replacement is ids[row][(v.y * n) >> 32], or (v.y * n_ent) >> 32 and one
//            miss when n = 0 (only the filter can empty a row).
// Both are deterministic: no atomics but the miss counter, and every stream depends on (seed, step, side, row, index) only.
#include <math.h>

#include "kge_rank_common.cuh"

namespace kge {

constexpr uint32_t NSC_KEY = 0x4E534341u;  // "NSCA": separates the refresh streams from the corruption / dropout / init ones
constexpr int NSC_THREADS = 128;

__device__ __forceinline__ uint32_t nsc_word(const NSCacheParams &p, long long row, unsigned idx, unsigned stream, int side)
{
    const u32x4 v = philox4x32_10((uint32_t)row, (idx >> 2) | (stream << 30) | ((unsigned)side << 31), (uint32_t)p.step,
                                  (uint32_t)(p.step >> 32), (uint32_t)p.seed, (uint32_t)(p.seed >> 32) ^ NSC_KEY);
    const unsigned w = idx & 3u;
    return w == 0 ? v.x : w == 1 ? v.y : w == 2 ? v.z : v.w;
}

// Column d (< kp) of the query vectors of one triple (s, p, o): os of side s (TransE p - o, DistMult p * o, ComplEx / HolE
// conj-rotated o, RotatE p's cos | sin with o's row in aux), oo of side o (s + p, s * p, s * p, the rotated subject).  s and
// o are the entity rows, prow the relation row's offset into rel (rot for RotatE), halves = model_halves(model).  The
// operations of kge_rank_qvec_kernel, one by one, so the scores are kge_corruption_scores'; a copy, because calling it
// from that kernel changes its SASS.
__device__ __forceinline__ void query_columns(int model, int halves, const float *__restrict__ s, const float *__restrict__ o,
                                              const float *__restrict__ rel, const float *__restrict__ rot, size_t prow,
                                              int d, int kp, float *os, float *oo, float *aux)
{
    if (halves == 1) {
        float p = rel[prow + d];
        if (model == KGE_TRANSE) { os[d] = __fsub_rn(p, o[d]); oo[d] = __fadd_rn(s[d], p); }
        else { os[d] = __fmul_rn(p, o[d]); oo[d] = __fmul_rn(s[d], p); }
    } else if (model == KGE_ROTATE) {
        float c = rot[prow + d], sn = rot[prow + kp + d];
        os[d] = c; os[kp + d] = sn;
        aux[d] = o[d]; aux[kp + d] = o[kp + d];
        oo[d] = __fmaf_rn(-s[kp + d], sn, __fmul_rn(s[d], c));
        oo[kp + d] = __fmaf_rn(s[kp + d], c, __fmul_rn(s[d], sn));
    } else {
        float pr = rel[prow + d], pi = rel[prow + kp + d];
        os[d] = __fmaf_rn(pi, o[kp + d], __fmul_rn(pr, o[d]));        // ComplEx.py:95-99
        os[kp + d] = __fmaf_rn(-pi, o[d], __fmul_rn(pr, o[kp + d]));   // ComplEx.py:101-106
        oo[d] = __fmaf_rn(-s[kp + d], pi, __fmul_rn(s[d], pr));        // ComplEx.py:139-143
        oo[kp + d] = __fmaf_rn(s[d], pi, __fmul_rn(s[kp + d], pr));    // ComplEx.py:145-149
    }
}

// The canonical score of candidate row e against the query q (a: the query's object row on RotatE's subject side): the
// ascending chain of pair_score_warp, read with 16-byte loads (ld and kp are multiples of 4)
template <int OP>
__device__ __forceinline__ float candidate_score(const float *__restrict__ e, const float *q, const float *a, int ld, int kp,
                                                 float scale)
{
    float acc = 0.f;
    if (OP != OP_ROT_S && OP != OP_ROT_O) {
        for (int d = 0; d < ld; d += 4) {
            const float4 ev = __ldg(reinterpret_cast<const float4 *>(e + d));
            const float4 qv = *reinterpret_cast<const float4 *>(q + d);
            acc = rank_step<OP>(acc, ev.x, qv.x);
            acc = rank_step<OP>(acc, ev.y, qv.y);
            acc = rank_step<OP>(acc, ev.z, qv.z);
            acc = rank_step<OP>(acc, ev.w, qv.w);
        }
    } else {
        for (int d = 0; d < kp; d += 4) {
            const float4 er = __ldg(reinterpret_cast<const float4 *>(e + d));
            const float4 ei = __ldg(reinterpret_cast<const float4 *>(e + kp + d));
            const float4 qr = *reinterpret_cast<const float4 *>(q + d), qi = *reinterpret_cast<const float4 *>(q + kp + d);
            float4 ar = make_float4(0.f, 0.f, 0.f, 0.f), ai = ar;
            if (OP == OP_ROT_S) { ar = *reinterpret_cast<const float4 *>(a + d); ai = *reinterpret_cast<const float4 *>(a + kp + d); }
            acc = rank_step_rot<OP>(acc, er.x, ei.x, qr.x, qi.x, ar.x, ai.x);
            acc = rank_step_rot<OP>(acc, er.y, ei.y, qr.y, qi.y, ar.y, ai.y);
            acc = rank_step_rot<OP>(acc, er.z, ei.z, qr.z, qi.z, ar.z, ai.z);
            acc = rank_step_rot<OP>(acc, er.w, ei.w, qr.w, qi.w, ar.w, ai.w);
        }
    }
    return rank_finish<OP>(acc, scale);
}

// OPS / OPO: the chains of the subject and object sides of the model (rank_op)
template <int OPS, int OPO>
__global__ void __launch_bounds__(NSC_THREADS) kge_nscaching_refresh_kernel(const NSCacheParams p)
{
    extern __shared__ __align__(16) float nsc_sm[];
    const int ld = p.ld, kp = p.kp, M = p.n1 + p.n2, t = threadIdx.x;
    float *qs = nsc_sm, *qo = qs + ld, *qa = qo + ld, *key = qa + ld;
    int *cid = reinterpret_cast<int *>(key + M);
    unsigned char *valid_c = reinterpret_cast<unsigned char *>(cid + M), *kept = valid_c + M;
    const long long items = 2 * p.B;
    for (long long w = blockIdx.x; w < items; w += gridDim.x) {
        if (!p.update[w]) continue;  // CTA-uniform
        const long long i = w >> 1;
        const int side = (int)(w & 1);
        const long long row = p.key_rows[w];
        const int s = p.triples[3 * i], rel = p.triples[3 * i + 1], o = p.triples[3 * i + 2];
        int32_t *ids = p.ids[side] + row * p.n1;
        const int n0 = p.count[side][row];
        const int m = n0 + p.n2;
        for (int d = t; d < kp; d += NSC_THREADS)
            query_columns(p.model, model_halves(p.model), p.ent + (size_t)s * ld, p.ent + (size_t)o * ld, p.rel, p.rel, (size_t)rel * ld, d, kp, qs, qo, qa);
        for (int c = t; c < m; c += NSC_THREADS)
            cid[c] = c < n0 ? ids[c] : (int)(((unsigned long long)nsc_word(p, row, (unsigned)(c - n0), 0, side) * p.n_ent) >> 32);
        __syncthreads();
        const long long fkey = (long long)rel * (long long)p.n_ent + (side ? s : o);
        for (int c = t; c < m; c += NSC_THREADS) {
            const int id = cid[c];
            bool valid = true;
            for (int c2 = 0; c2 < c && valid; ++c2) valid = cid[c2] != id;
            if (valid && p.filt_n[side] > 0) valid = !known_pair(p.filt_keys[side], p.filt_vals[side], p.filt_n[side], fkey, id);
            float k = 0.f;
            if (valid) {
                const float *e = p.ent + (size_t)id * ld;
                const float sc = side ? candidate_score<OPO>(e, qo, nullptr, ld, kp, p.scale) : candidate_score<OPS>(e, qs, qa, ld, kp, p.scale);
                valid = !isnan(sc);
                const float u = ((float)(nsc_word(p, row, (unsigned)c, 1, side) >> 9) + 0.5f) * 0x1p-23f;
                k = __fadd_rn(sc, -logf(-logf(u)));
            }
            key[c] = k;
            valid_c[c] = valid;
        }
        __syncthreads();
        // rank among the valid candidates: (larger key, then lower c) first; the first N1 are kept
        for (int c = t; c < m; c += NSC_THREADS) {
            int r = 0;
            if (valid_c[c]) {
                const float k = key[c];
                for (int c2 = 0; c2 < m; ++c2) r += valid_c[c2] && (key[c2] > k || (key[c2] == k && c2 < c));
            }
            kept[c] = valid_c[c] && r < p.n1;
        }
        __syncthreads();
        for (int c = t; c < m; c += NSC_THREADS) {
            if (!kept[c]) continue;
            int pos = 0;
            for (int c2 = 0; c2 < c; ++c2) pos += kept[c2];
            ids[pos] = cid[c];
        }
        if (t == 0) {  // every thread read the old count before the first barrier
            int n = 0;
            for (int c = 0; c < m; ++c) n += kept[c];
            p.count[side][row] = n;
        }
        __syncthreads();  // the shared arrays are reused by the CTA's next item
    }
}

__global__ void __launch_bounds__(256) kge_nscaching_draw_kernel(const NSCacheParams p)
{
    const unsigned long long n = (unsigned long long)p.B * (unsigned long long)p.eta;
    const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
    for (unsigned long long r = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += stride) {
        const long long i = (long long)(r % (unsigned long long)p.B);
        const u32x4 v = philox4x32_10((uint32_t)r, (uint32_t)(r >> 32), (uint32_t)p.step, (uint32_t)(p.step >> 32),
                                      (uint32_t)p.seed, (uint32_t)(p.seed >> 32));
        const int side = (int)(v.x & 1u);
        const long long row = p.key_rows[2 * i + side];
        const unsigned cnt = (unsigned)p.count[side][row];
        int c;
        if (cnt > 0) {
            c = p.ids[side][row * p.n1 + (long long)(((unsigned long long)v.y * cnt) >> 32)];
        } else {
            c = (int)(((unsigned long long)v.y * p.n_ent) >> 32);
            if (p.misses) atomicAdd(p.misses, 1ull);
        }
        p.neg_ent[r] = c;
        p.neg_keep[r] = (uint8_t)side;
    }
}

size_t nscaching_smem_bytes(int ld, int n1, int n2)
{
    const int m = n1 + n2;
    return (size_t)(3 * ld + m) * sizeof(float) + (size_t)m * sizeof(int) + 2 * (size_t)m;
}

cudaError_t launch_nscaching(const NSCacheParams &p, int sm_count, cudaStream_t st)
{
    if (p.B == 0) return cudaSuccess;
    const long long items = 2 * p.B, cap = 16ll * sm_count;
    const unsigned grid = (unsigned)(items < cap ? items : cap);
    const size_t smem = nscaching_smem_bytes(p.ld, p.n1, p.n2);
    cudaError_t e;
    if (p.model == KGE_TRANSE)
        e = launch_with_smem(kge_nscaching_refresh_kernel<OP_L1_ADD, OP_L1_SUB>, grid, NSC_THREADS, smem, st, p);
    else if (p.model == KGE_ROTATE)
        e = launch_with_smem(kge_nscaching_refresh_kernel<OP_ROT_S, OP_ROT_O>, grid, NSC_THREADS, smem, st, p);
    else
        e = launch_with_smem(kge_nscaching_refresh_kernel<OP_DOT, OP_DOT>, grid, NSC_THREADS, smem, st, p);
    if (e != cudaSuccess) return e;
    const long long n = p.B * (long long)p.eta;
    const long long want = (n + 255) / 256, dcap = 16ll * sm_count;
    kge_nscaching_draw_kernel<<<(unsigned)(want < dcap ? want : dcap), 256, 0, st>>>(p);
    return cudaGetLastError();
}

}  // namespace kge
