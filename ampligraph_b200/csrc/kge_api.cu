// kge_api.cu -- the extern "C" boundary of libkge_b200.so (see include/kge_b200.h).
#include <float.h>
#include <stdarg.h>
#include <stddef.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <new>

#include "kge_internal.h"
#include "kge_optim_common.cuh"  // uses_slot0 / uses_slot1: which slot buffers a kind needs
#include "kge_rank_common.cuh"  // the OP_* chains kge_knn / kge_radius_neighbors choose by metric

using namespace kge;

// the training kernels, each with its own slot geometry (kge_handle::slot)
enum TrainPath {
    TRAIN_GENERAL,  // kge_train.cu: any shape
    TRAIN_RES,      // kge_train_res.cu: the resident trilinear fast path
    TRAIN_ROT,      // kge_train_rot.cu: the RotatE fast path
    TRAIN_PATHS
};

struct kge_handle {
    kge_config cfg;
    Layout L;
    int sm_count;
    int max_smem;
    float score_scale;  // HolE 2/k
    float rot_div;      // RotatE range/pi
    // the only device memory the library owns (allocated once by kge_create, freed by kge_destroy):
    float *rot;              // [n_rel, ld] rotation table (RotatE only)
    unsigned *done_counter;  // [0]: last-CTA counter of kge_optimizer_step_exchange; [1], [2]: the training kernels' positive counter and retired-warp counter (self-resetting)
    unsigned long long *exchange_trace;  // caller-owned 8 x uint64 phase stamps of the next exchange launches, or nullptr
    // training launch geometry: the row layout every kernel shares, then one slot per kernel
    int nit, eta_pad, wk, n_cb, slot_floats;
    int nbuf, resident;  // the general kernel's group buffers and residency (kge_rows_resident)
    TrainSlot slot[TRAIN_PATHS];
    int *stamp_ent, *stamp_rel;  // lazy-optimizer row stamps (caller-owned) or nullptr
    float *stash;                // caller-owned row stash for sharded runs (kge_set_row_stash) or nullptr
    long long stash_rows;
    int hot_ent[2];              // kge_set_hot_entities (-1: none)
    int l2_bytes;                // cudaDeviceProp::l2CacheSize
    long long topk_chunk;        // KGE_B200_TOPK_CHUNK: candidates per kge_topk chunk (0: sized to L2)
    void *train_ws;              // caller-owned training workspace (kge_set_train_workspace) or nullptr
    long long train_ws_bytes;
    // KGE_STEP_FUSED_DEFER: the step whose replaced-row sum waits in the workspace for kge_optimizer_step_deferred
    bool sum_pending;
    TrainParams pending;
    // kge_set_embedding_dropout: the all-candidate steps' embedding dropout (both 0: none)
    float drop_p_ent, drop_p_rel;
    uint64_t drop_seed;
};

// Make the handle's device current for the duration of an entry point (ADVICE r1: two handles on different GPUs
// driven from one thread); restores the caller's device on return.
struct DeviceGuard {
    int prev = -1;
    bool switched = false;
    cudaError_t err = cudaSuccess;
    explicit DeviceGuard(int dev)
    {
        err = cudaGetDevice(&prev);
        if (err == cudaSuccess && prev != dev) {
            err = cudaSetDevice(dev);
            switched = err == cudaSuccess;
        }
    }
    ~DeviceGuard()
    {
        if (switched) cudaSetDevice(prev);
    }
};
#define KGE_GUARD(h)                       \
    DeviceGuard guard_((h)->cfg.device);   \
    if (guard_.err != cudaSuccess) return cuda_fail(guard_.err, "cudaSetDevice")

static thread_local char g_err[512] = "";

static int fail(int code, const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}
static int cuda_fail(cudaError_t e, const char *what)
{
    return fail(KGE_ERR_CUDA, "%s: %s (%s)", what, cudaGetErrorName(e), cudaGetErrorString(e));
}
#define KGE_CUDA(call, what)                                 \
    do {                                                     \
        cudaError_t e_ = (call);                             \
        if (e_ != cudaSuccess) return cuda_fail(e_, what);   \
    } while (0)

extern "C" const char *kge_last_error(void) { return g_err; }
extern "C" int kge_abi_version(void) { return KGE_B200_ABI_VERSION; }

extern "C" int kge_create(const kge_config *cfg, kge_handle **out)
{
    if (!cfg || !out) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_create: null argument");
    if (cfg->struct_size != (int32_t)sizeof(kge_config))
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_create: kge_config.struct_size %d != %d (ABI mismatch)",
                    cfg->struct_size, (int)sizeof(kge_config));
    if (cfg->scoring < KGE_TRANSE || cfg->scoring > KGE_ROTATE)
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_create: unknown scoring_type id %d", cfg->scoring);
    if (cfg->loss < KGE_LOSS_PAIRWISE || cfg->loss > KGE_LOSS_MULTICLASS_NLL)
        return fail(KGE_ERR_INVALID_ARGUMENT, "Could not interpret loss identifier: %d", cfg->loss);
    if (cfg->reduction != KGE_REDUCE_SUM && cfg->reduction != KGE_REDUCE_MEAN)
        return fail(KGE_ERR_INVALID_ARGUMENT, "Invalid value for reduction!");
    if (cfg->rank_mode != KGE_RANK_MODE_AUTO && cfg->rank_mode != KGE_RANK_MODE_EXACT)
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_create: unknown rank_mode %d", cfg->rank_mode);
    if (cfg->max_rel_size < 0 || cfg->rank_pair_cap < 0) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_create: max_rel_size / rank_pair_cap < 0");
    if (cfg->k < 1 || cfg->eta < 1 || cfg->n_ent < 1 || cfg->n_rel < 1)
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_create: k, eta, n_ent, n_rel must be >= 1");
    if (cfg->n_ent > 0x7fffffffLL || cfg->n_rel > 0x7fffffffLL)
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_create: ids are int32 (n_ent, n_rel < 2^31)");

    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return fail(KGE_ERR_CUDA, "kge_create: no CUDA device visible (%s) -- libkge_b200 has no CPU path",
                    e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
    if (cfg->device < 0 || cfg->device >= ndev)
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_create: device %d out of range [0,%d)", cfg->device, ndev);
    DeviceGuard guard_(cfg->device);
    if (guard_.err != cudaSuccess) return cuda_fail(guard_.err, "cudaSetDevice");
    cudaDeviceProp prop;
    KGE_CUDA(cudaGetDeviceProperties(&prop, cfg->device), "cudaGetDeviceProperties");
    if (prop.major != 9 || prop.minor != 0)
        return fail(KGE_ERR_UNSUPPORTED, "kge_create: device is sm_%d%d; libkge_b200 is built for sm_90a only",
                    prop.major, prop.minor);

    kge_handle *h = new (std::nothrow) kge_handle();
    if (!h) return fail(KGE_ERR_CUDA, "kge_create: out of host memory");
    memset(h, 0, sizeof(*h));
    h->cfg = *cfg;
    Layout &L = h->L;
    L.model = cfg->scoring;
    L.k = cfg->k;
    L.halves = model_halves(cfg->scoring);
    L.kp = (cfg->k + 3) / 4 * 4;
    L.ld = L.halves * L.kp;
    L.K = L.halves * cfg->k;
    h->sm_count = prop.multiProcessorCount;
    h->max_smem = (int)prop.sharedMemPerBlockOptin;
    h->l2_bytes = prop.l2CacheSize;
    // development switch: force the kge_topk chunk (the tests use it to run many chunks over small tables)
    if (const char *ev = getenv("KGE_B200_TOPK_CHUNK")) { const long long c = atoll(ev); if (c >= 1) h->topk_chunk = c; }
    h->score_scale = (cfg->scoring == KGE_HOLE) ? hole_scale(L.K) : 1.f;
    h->rot_div = (cfg->scoring == KGE_ROTATE) ? rotate_divisor(L.K, cfg->max_rel_size > 0 ? cfg->max_rel_size : cfg->n_rel) : 1.f;

    // ---- training geometry: one warp per positive; its slot holds (3+G) row windows ----
    // window = wk floats per half (<= 128*NIT so that NIT float4 per lane cover it); rows wider than
    // 512 floats per half are processed in n_cb column windows, eta > G negatives in groups of G.
    const int nch = L.kp / 4;
    const int nit_raw = (nch + 31) / 32;
    h->nit = nit_raw <= 1 ? 1 : nit_raw <= 2 ? 2 : 4;
    h->wk = L.kp <= 512 ? L.kp : 512;
    h->n_cb = (L.kp + h->wk - 1) / h->wk;
    h->eta_pad = (cfg->eta + 3) / 4 * 4;
    const int row_bytes = L.halves * h->wk * 4, aux = 4 * h->eta_pad * 4 + 16;  // sc | nid | nside | jorig, two mbarriers
    h->slot_floats = row_bytes / 4;
    int max_warps = KGE_TRAIN_THREADS(cfg->scoring, h->nit) / 32;
    int nbuf = 2;  // group buffers of a non-resident slot
    // tuning aids (scripts/kbench.py): cap the warps per CTA, choose the buffering of non-resident slots
    if (const char *ev = getenv("KGE_B200_TRAIN_WARPS")) { const int w = atoi(ev); if (w >= 1 && w < max_warps) max_warps = w; }
    if (const char *ev = getenv("KGE_B200_TRAIN_NBUF")) nbuf = atoi(ev) == 1 ? 1 : 2;
    // Residency policy (scripts/kbench.py sweeps run before the H100 port; not re-run): keep all eta corruptions resident
    // (one gather per row) while >= KGE_MIN_RESIDENT_WARPS warps still fit; otherwise shrink G until
    // min(max_warps, KGE_TARGET_WARPS) warps fit -- the gradient pass then re-gathers the other groups, which
    // costs less than running with few warps.
    // non-resident slots hold TWO group buffers (the next group is prefetched while the current one is processed)
    int G = cfg->eta;
    bool res = h->n_cb == 1;
    if (cfg->neg_group > 0) {
        G = cfg->neg_group < cfg->eta ? cfg->neg_group : cfg->eta;
        res = res && G >= cfg->eta;
    } else {
        const long long full = (3 + (long long)cfg->eta) * row_bytes + aux;
        const int min_res = max_warps < KGE_MIN_RESIDENT_WARPS ? max_warps : KGE_MIN_RESIDENT_WARPS;
        if (!res || full * min_res > h->max_smem) {
            res = false;
            const int want = max_warps < KGE_TARGET_WARPS ? max_warps : KGE_TARGET_WARPS;
            while (G > 1 && (long long)((3 + nbuf * G) * (long long)row_bytes + aux) * want > h->max_smem) --G;
        }
    }
    h->resident = res ? 1 : 0;
    h->nbuf = nbuf;
    {
        const int rows = (res ? 3 + G : 3 + nbuf * G) * row_bytes, region = rows + aux;
        const int warps = h->max_smem / region;  // 0 => even (3+1) windows do not fit (reported by kge_train_step)
        h->slot[TRAIN_GENERAL] = {warps < max_warps ? warps : max_warps, G, rows, region};
    }
    h->hot_ent[0] = h->hot_ent[1] = -1;

    // ---- the resident trilinear fast path (kge_train_res.cu): DistMult / ComplEx / HolE, one window, eta <= 32; its slot
    // holds s, o and the eta replaced rows (the relation row lives in registers) + sc | nid | jorig + one mbarrier.
    // Same residency rule as above, with its own (one row smaller) slot.
    // DistMult rows of up to 512 floats (NIT = 4) qualify too: its per-lane state is a third of ComplEx's.
    if ((cfg->scoring == KGE_DISTMULT || cfg->scoring == KGE_COMPLEX || cfg->scoring == KGE_HOLE) && h->n_cb == 1 &&
        (h->nit <= 2 || cfg->scoring == KGE_DISTMULT) && cfg->eta <= 32 && cfg->neg_group <= 0) {
        const int rows = (2 + cfg->eta) * row_bytes, region = rows + (3 * h->eta_pad * 4 + 8 + 15) / 16 * 16;
        int rw = h->max_smem / region;
        if (rw > max_warps) rw = max_warps;
        int min_res = max_warps < KGE_MIN_RESIDENT_WARPS ? max_warps : KGE_MIN_RESIDENT_WARPS;
        if (h->nit == 4) min_res = KGE_MIN_RESIDENT_WARPS_WIDE;
        if (const char *ev = getenv("KGE_B200_RES_MIN_WARPS")) min_res = atoi(ev);  // tuning aid
        if (rw >= min_res) h->slot[TRAIN_RES] = {rw, cfg->eta, rows, region};
    }

    // ---- the RotatE fast path (kge_train_rot.cu): one window, rows of up to 256 floats per half; its slot holds ONLY replaced
    // rows (s, o and the rotation row live in registers): all eta of them when they fit beside 8 warps, else two buffers of G.
    if (cfg->scoring == KGE_ROTATE && h->n_cb == 1 && h->nit <= 2 && cfg->neg_group <= 0) {
        const int rot_aux = (4 * h->eta_pad * 4 + 16 + 15) / 16 * 16;  // sc | nid | jorig | side, two mbarriers
        const int rw = 8;                                                // 256 threads (launch bound of the kernel)
        const int cap = (h->max_smem / rw - rot_aux) / row_bytes;        // rows per warp
        int rG = cap >= cfg->eta ? cfg->eta : cap / 2;
        if (const char *ev = getenv("KGE_B200_ROT_G")) {  // tuning aid: smaller groups
            const int g = atoi(ev);
            if (g >= 1 && g <= cap / 2 && g < cfg->eta) rG = g;
        }
        const int rows = (rG >= cfg->eta ? rG : 2 * rG) * row_bytes;
        if (rG >= 1) h->slot[TRAIN_ROT] = {rw, rG, rows, rows + rot_aux};
    }

    if (cfg->scoring == KGE_ROTATE) {
        cudaError_t e2 = cudaMalloc(&h->rot, (size_t)cfg->n_rel * L.ld * sizeof(float));
        if (e2 != cudaSuccess) { delete h; return cuda_fail(e2, "cudaMalloc(rotation table)"); }
    }
    {
        cudaError_t e2 = cudaMalloc(&h->done_counter, 4 * sizeof(unsigned));
        if (e2 == cudaSuccess) e2 = cudaMemset(h->done_counter, 0, 4 * sizeof(unsigned));
        if (e2 != cudaSuccess) { if (h->rot) cudaFree(h->rot); delete h; return cuda_fail(e2, "cudaMalloc(counter)"); }
    }
    *out = h;
    return KGE_OK;
}

extern "C" void kge_destroy(kge_handle *h)
{
    if (!h) return;
    DeviceGuard guard_(h->cfg.device);
    if (h->rot) cudaFree(h->rot);
    if (h->done_counter) cudaFree(h->done_counter);
    delete h;
}

extern "C" int32_t kge_internal_k(const kge_handle *h) { return h ? h->L.K : 0; }
extern "C" int32_t kge_half_stride(const kge_handle *h) { return h ? h->L.kp : 0; }
extern "C" int32_t kge_row_stride(const kge_handle *h) { return h ? h->L.ld : 0; }

// null check + device guard (every entry point below launches on the handle's device)
#define KGE_CHECK_HANDLE(h, fn)                                           \
    if (!(h)) return fail(KGE_ERR_INVALID_ARGUMENT, fn ": null handle"); \
    KGE_GUARD(h)

extern "C" int kge_pack_rows(kge_handle *h, const float *dense_dev, float *table_dev, int64_t rows, void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_pack_rows");
    if (rows < 0 || (rows > 0 && (!dense_dev || !table_dev))) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_pack_rows: bad argument");
    KGE_CUDA(launch_pack(h->L, dense_dev, table_dev, rows, false, (cudaStream_t)stream), "kge_pack_rows");
    return KGE_OK;
}
extern "C" int kge_unpack_rows(kge_handle *h, const float *table_dev, float *dense_dev, int64_t rows, void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_unpack_rows");
    if (rows < 0 || (rows > 0 && (!dense_dev || !table_dev))) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_unpack_rows: bad argument");
    KGE_CUDA(launch_pack(h->L, table_dev, dense_dev, rows, true, (cudaStream_t)stream), "kge_unpack_rows");
    return KGE_OK;
}

extern "C" int kge_init_glorot_uniform(kge_handle *h, float *table_dev, int64_t rows, uint64_t seed, void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_init_glorot_uniform");
    if (rows < 0 || (rows > 0 && !table_dev)) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_init_glorot_uniform: bad argument");
    KGE_CUDA(launch_glorot(h->L, table_dev, rows, seed, (cudaStream_t)stream), "kge_init_glorot_uniform");
    return KGE_OK;
}

extern "C" int kge_init_table(kge_handle *h, float *table_dev, int64_t rows, int32_t kind, float a, float b, uint64_t seed,
                              void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_init_table");
    if (rows < 0 || (rows > 0 && !table_dev)) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_init_table: bad argument");
    if (kind < KGE_INIT_UNIFORM || kind > KGE_INIT_CONSTANT) return fail(KGE_ERR_INVALID_ARGUMENT, "Unknown initializer kind: %d", kind);
    if ((kind == KGE_INIT_NORMAL || kind == KGE_INIT_TRUNCATED_NORMAL) && b < 0.f)
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_init_table: negative stddev");
    KGE_CUDA(launch_init_table(h->L, table_dev, rows, kind, a, b, seed, (cudaStream_t)stream), "kge_init_table");
    return KGE_OK;
}

static int refresh_rotation(kge_handle *h, const float *rel_dev, cudaStream_t st)
{
    if (h->cfg.scoring != KGE_ROTATE) return KGE_OK;
    KGE_CUDA(launch_rotation_table(rel_dev, h->rot, h->cfg.n_rel, h->L.kp, h->L.ld, h->rot_div, st),
             "rotation table");
    return KGE_OK;
}

// The relation rows a step or query reads: for RotatE the rotation table refresh_rotation writes, else the relation table
static const float *relation_rows(const kge_handle *h, const float *rel_dev)
{
    return h->cfg.scoring == KGE_ROTATE ? h->rot : rel_dev;
}

extern "C" int kge_score_triples(kge_handle *h, const float *ent_dev, const float *rel_dev,
                                 const int32_t *triples_dev, int64_t n, float *scores_dev, void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_score_triples");
    if (n < 0) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_score_triples: n < 0");
    if (n == 0) return KGE_OK;
    if (!ent_dev || !rel_dev || !triples_dev || !scores_dev)
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_score_triples: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    if (int rc = refresh_rotation(h, rel_dev, st)) return rc;
    KGE_CUDA(launch_score_triples(h->L, h->nit, ent_dev, relation_rows(h, rel_dev), triples_dev, n, h->score_scale,
                                  scores_dev, h->sm_count, st),
             "kge_score_triples");
    return KGE_OK;
}

extern "C" int kge_generate_corruptions(kge_handle *h, const int32_t *triples_dev, int64_t B, uint64_t seed,
                                        uint64_t step, int32_t *corruptions_dev, void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_generate_corruptions");
    if (B < 0) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_generate_corruptions: B < 0");
    if (B == 0) return KGE_OK;
    if (!triples_dev || !corruptions_dev) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_generate_corruptions: null pointer");
    KGE_CUDA(launch_corruptions(triples_dev, B, h->cfg.eta, seed, step, (unsigned)h->cfg.n_ent, corruptions_dev,
                                (cudaStream_t)stream),
             "kge_generate_corruptions");
    return KGE_OK;
}

// ---- the sampled steps' shared checks and set-up: the negative sampler, NSCaching, shared negatives, the fused step ----

// A kge_negative_sampler's header: its struct_size, and max_attempts 1..256 (the attempt is the top byte of the Philox
// counter's second word)
static int check_sampler(const kge_negative_sampler *q, const char *fn)
{
    if (!q || q->struct_size != (int32_t)sizeof(kge_negative_sampler) || q->max_attempts < 1 || q->max_attempts > 256)
        return fail(KGE_ERR_INVALID_ARGUMENT, "%s: bad kge_negative_sampler (ABI mismatch or max_attempts outside 1..256)",
                    fn);
    return KGE_OK;
}

// The known-pair filter of both sides of a sampler struct (kge_negative_sampler, kge_nscaching): refuses a count < 0,
// or > 0 without its arrays, and copies them into the filt_* arrays of the launch parameters p (NegativeParams,
// NSCacheParams; [0] a replaced subject, [1] a replaced object).  The kernels keep three arrays rather than one struct per
// side: indexing a struct by side costs the NSCaching refresh kernels up to 10 registers.
template <class Sampler, class Params> static int side_filters(const Sampler *q, const char *fn, Params &p)
{
    p.filt_n[0] = q->sub_filter_n;
    p.filt_keys[0] = reinterpret_cast<const long long *>(q->sub_filter_keys_dev);
    p.filt_vals[0] = q->sub_filter_vals_dev;
    p.filt_n[1] = q->obj_filter_n;
    p.filt_keys[1] = reinterpret_cast<const long long *>(q->obj_filter_keys_dev);
    p.filt_vals[1] = q->obj_filter_vals_dev;
    for (int side = 0; side < 2; ++side)
        if (p.filt_n[side] < 0 || (p.filt_n[side] > 0 && (!p.filt_keys[side] || !p.filt_vals[side])))
            return fail(KGE_ERR_INVALID_ARGUMENT, "%s: a filter count < 0, or > 0 without its arrays", fn);
    return KGE_OK;
}

// A sampled batch of B positives: B >= 0 and eta*B < 2^56 (corruption r = j*B + i shares a Philox counter word with
// the sampler's attempt byte)
static int check_sampled_batch(const kge_handle *h, int64_t B, const char *fn)
{
    if (B < 0) return fail(KGE_ERR_INVALID_ARGUMENT, "%s: B < 0", fn);
    if (B > ((1ll << 56) - 1) / h->cfg.eta) return fail(KGE_ERR_INVALID_ARGUMENT, "%s: eta*B >= 2^56", fn);
    return KGE_OK;
}

// The steps that read one whole entity table (NSCaching, shared negatives) refuse while a row stash is set
static int check_no_stash(const kge_handle *h, const char *fn)
{
    if (h->stash)
        return fail(KGE_ERR_UNSUPPORTED, "%s: a row stash is set (row-sharded tables), and this step reads one whole "
                                         "entity table", fn);
    return KGE_OK;
}

static bool dropout_set(const kge_handle *h) { return h->drop_p_ent != 0.f || h->drop_p_rel != 0.f; }

// The sampled steps' fused kernels read the raw rows: they refuse while embedding dropout is set
static int check_no_dropout(const kge_handle *h, const char *fn)
{
    if (!dropout_set(h)) return KGE_OK;
    return fail(KGE_ERR_UNSUPPORTED, "%s: embedding dropout is set (kge_set_embedding_dropout), and the sampled training "
                                     "kernels do not apply it: it applies to kge_one_vs_all_step, "
                                     "kge_one_vs_all_relation_step and kge_k_vs_all_step; clear it with (0, 0)", fn);
}

// The TrainParams of a sampled training step that come from the handle and the call: the tables (rel as relation_rows
// gives it: refresh_rotation first), the triples, the Philox key, the row shape, the loss and the lazy-optimizer
// stamps.  Every other field is zero.  The kernels write the relation stamps only while the entity stamps are set.
static TrainParams sampled_train_params(const kge_handle *h, const float *ent_dev, const float *rel_dev,
                                        float *grad_ent_dev, float *grad_rel_dev, const int32_t *triples_dev, int64_t B,
                                        uint64_t seed, uint64_t step, double *loss_dev)
{
    TrainParams p;
    memset(&p, 0, sizeof(p));
    p.ent = ent_dev;
    p.rel = relation_rows(h, rel_dev);
    p.grad_ent = grad_ent_dev;
    p.grad_rel = grad_rel_dev;
    p.triples = triples_dev;
    p.B = B;
    p.seed = seed;
    p.step = step;
    p.n_ent = (unsigned)h->cfg.n_ent;
    p.model = h->cfg.scoring;
    p.eta = h->cfg.eta;
    p.kp = h->L.kp;
    p.ld = h->L.ld;
    p.nch = h->L.kp / 4;
    p.loss = h->cfg.loss;
    p.reduction = h->cfg.reduction;
    p.margin = h->cfg.margin;
    p.alpha = h->cfg.alpha;
    p.score_scale = h->score_scale;
    p.inv_div = 1.f / h->rot_div;
    p.loss_out = loss_dev;
    p.stamp = kge_step_stamp(step);
    p.stamp_ent = h->stamp_ent;
    p.stamp_rel = h->stamp_rel;
    return p;
}

extern "C" int kge_sample_negatives(kge_handle *h, const kge_negative_sampler *sampler, const int32_t *triples_dev,
                                    int64_t B, uint64_t seed, uint64_t step, int32_t *neg_ent_dev,
                                    uint8_t *neg_keep_subj_dev, uint64_t *misses_dev, void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_sample_negatives");
    const kge_negative_sampler *q = sampler;
    if (int rc = check_sampler(q, "kge_sample_negatives")) return rc;
    if ((q->sub_pool_off_dev == nullptr) != (q->sub_pool_ids_dev == nullptr) ||
        (q->obj_pool_off_dev == nullptr) != (q->obj_pool_ids_dev == nullptr))
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_sample_negatives: a pool needs both its offsets and its ids");
    NegativeParams p;
    memset(&p, 0, sizeof(p));
    if (int rc = side_filters(q, "kge_sample_negatives", p)) return rc;
    if (int rc = check_sampled_batch(h, B, "kge_sample_negatives")) return rc;
    if (B == 0) return KGE_OK;
    if (!triples_dev || !neg_ent_dev || !neg_keep_subj_dev)
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_sample_negatives: null triples or output pointer");
    p.triples = triples_dev;
    p.B = B;
    p.eta = h->cfg.eta;
    p.max_attempts = q->max_attempts;
    p.n_ent = (unsigned)h->cfg.n_ent;
    p.seed = seed;
    p.step = step;
    p.thr = q->thresholds_dev;
    p.pool_off[0] = reinterpret_cast<const long long *>(q->sub_pool_off_dev);
    p.pool_ids[0] = q->sub_pool_ids_dev;
    p.pool_off[1] = reinterpret_cast<const long long *>(q->obj_pool_off_dev);
    p.pool_ids[1] = q->obj_pool_ids_dev;
    p.neg_ent = neg_ent_dev;
    p.neg_keep = neg_keep_subj_dev;
    p.misses = reinterpret_cast<unsigned long long *>(misses_dev);
    KGE_CUDA(launch_negatives(p, h->sm_count, (cudaStream_t)stream), "kge_sample_negatives");
    return KGE_OK;
}

// ---- host-side replay of the corruption stream (no GPU, no handle) -----------------------------------------
extern "C" void kge_philox4x32_10(const uint32_t ctr[4], const uint32_t key[2], uint32_t out[4])
{
    const u32x4 v = philox4x32_10(ctr[0], ctr[1], ctr[2], ctr[3], key[0], key[1]);
    out[0] = v.x; out[1] = v.y; out[2] = v.z; out[3] = v.w;
}

extern "C" int kge_host_corruptions(const int32_t *triples_host, int64_t B, int32_t eta, int64_t n_ent, uint64_t seed,
                                    uint64_t step, int32_t *corruptions_host)
{
    if (B < 0 || eta < 1 || n_ent < 1 || n_ent > 0x7fffffffLL)
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_host_corruptions: need B >= 0, eta >= 1, 1 <= n_ent < 2^31");
    if (B == 0) return KGE_OK;
    if (!triples_host || !corruptions_host) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_host_corruptions: null pointer");
    for (int64_t r = 0; r < B * (int64_t)eta; ++r) {  // same draw, same row order as kge_corruptions_kernel
        const int64_t i = r % B;
        int keep, repl;
        draw_corruption(seed, step, (unsigned long long)r, (uint32_t)n_ent, &keep, &repl);
        corruptions_host[3 * r + 0] = keep ? triples_host[3 * i + 0] : repl;
        corruptions_host[3 * r + 1] = triples_host[3 * i + 1];
        corruptions_host[3 * r + 2] = keep ? repl : triples_host[3 * i + 2];
    }
    return KGE_OK;
}

static int check_shard_map(const kge_handle *h, const kge_shard_map *map, const char *fn)
{
    if (!map || map->struct_size != (int32_t)sizeof(kge_shard_map))
        return fail(KGE_ERR_INVALID_ARGUMENT, "%s: bad kge_shard_map (ABI mismatch)", fn);
    if (map->world < 1 || map->world > KGE_MAX_PEERS || map->rows_per_shard < 1)
        return fail(KGE_ERR_INVALID_ARGUMENT, "%s: world must be 1..%d, rows_per_shard >= 1", fn, KGE_MAX_PEERS);
    if (map->rows_per_shard * (int64_t)map->world < h->cfg.n_ent)
        return fail(KGE_ERR_INVALID_ARGUMENT, "%s: world*rows_per_shard < n_ent", fn);
    for (int q = 0; q < map->world; ++q)
        if (!map->ent[q]) return fail(KGE_ERR_INVALID_ARGUMENT, "%s: null entity shard pointer for rank %d", fn, q);
    return KGE_OK;
}

// Bump allocation of a caller-owned workspace: each region starts at a multiple of its alignment and is padded to one;
// `at` is the bytes taken so far.  base == nullptr only sizes the workspace (every region is then nullptr).
struct Carve {
    char *base;
    size_t at = 0;
    explicit Carve(void *ws) : base(static_cast<char *>(ws)) {}
    template <class T> T *take(size_t bytes, size_t align)
    {
        at = (at + align - 1) / align * align;
        T *q = base ? reinterpret_cast<T *>(base + at) : nullptr;
        at += (bytes + align - 1) / align * align;
        return q;
    }
};

// Carve-up of the training workspace for a batch of B positives (the owner-computes path of the resident kernel,
// kge_train_bucket.cu): the per-entity counts first, so that they stay where kge_set_train_workspace zeroed them whatever B is.
static TrainParams::Buckets carve_train_workspace(const kge_handle *h, int64_t B, Carve &c)
{
    const size_t E = h->cfg.n_ent, n = (size_t)h->cfg.eta * B;
    TrainParams::Buckets bk;
    bk.cnt = c.take<int>(4 * E, 16);
    bk.off = c.take<int>(4 * (E + 1), 16);
    bk.tiles = c.take<int>(4 * ((E + 8191) / 8192), 16);
    bk.pos = c.take<int>(4 * n, 16);
    bk.eid = c.take<int>(4 * n, 16);
    bk.other = c.take<int>(4 * n, 16);
    bk.rel = c.take<int>(4 * n, 16);
    bk.g = c.take<float>(4 * n, 16);
    return bk;
}

// The caller's row stash, where it holds the eta*B replaced rows of a step of B positives (kge_set_row_stash), else nullptr.
static float *row_stash(const kge_handle *h, int64_t B)
{
    return (h->stash && h->stash_rows >= B * (int64_t)h->cfg.eta) ? h->stash : nullptr;
}

// The kernel a training step runs: a fast path where its slot applies, on one (not row-sharded) table and without a row
// stash; the general kernel otherwise, and for every shape under KGE_B200_TRAIN_KERNEL=general (A/B runs, and the tests
// that cover its resident trilinear instantiations).
static TrainPath train_path(const kge_handle *h, const kge_shard_map *map, const float *stash)
{
    const char *force = getenv("KGE_B200_TRAIN_KERNEL");
    if ((map && map->world > 1) || stash || (force && strcmp(force, "general") == 0)) return TRAIN_GENERAL;
    if (h->slot[TRAIN_ROT].warps > 0) return TRAIN_ROT;
    if (h->slot[TRAIN_RES].warps > 0) return TRAIN_RES;
    return TRAIN_GENERAL;
}

// Bytes of training workspace the owner-computes path needs for a step of B positives, or 0 where it does not apply: it
// applies where an unsharded step runs the resident kernel (train_path: not under KGE_B200_TRAIN_KERNEL=general, not with
// a row stash), the step replaces every entity at least once on average (eta*B >= n_ent), the entries fit int32 offsets
// (eta*B < 2^31), and KGE_B200_TRAIN_REPL=scatter (A/B runs, the tests that compare the two) does not keep the REDs.  This is
// the one place that decides whether a step buckets: kge_train_step gathers exactly when this is > 0 and the workspace set
// holds it, and callers decide from it whether a step can be deferred (KGE_STEP_FUSED_DEFER).  The bucket sum reads one
// kept-side entity row per corruption; it pays where replaced entities repeat within a step (measured on H100: cfg2, 19
// corruptions per entity, and cfg3, 4.2, gain) and loses where they do not ('big' in scripts/kbench.py: 2 M entities, 0.33
// per entity, HBM-resident, 1.65 -> 1.88 ms; DESIGN.md 5).
static int64_t bucket_workspace_bytes(const kge_handle *h, int64_t B)
{
    const char *rv = getenv("KGE_B200_TRAIN_REPL");
    const long long n = (long long)h->cfg.eta * B;
    if (train_path(h, nullptr, row_stash(h, B)) != TRAIN_RES || n < h->cfg.n_ent || n >= (1ll << 31) ||
        (rv && strcmp(rv, "scatter") == 0))
        return 0;
    Carve c(nullptr);
    carve_train_workspace(h, B, c);
    return (int64_t)c.at;
}

extern "C" int64_t kge_train_workspace_bytes(const kge_handle *h, int64_t B)
{
    return h && B >= 0 ? bucket_workspace_bytes(h, B) : 0;
}

// A KGE_STEP_FUSED_DEFER step leaves its replaced-row sum in the training workspace until kge_optimizer_step_deferred
// consumes it: until then no call may train or replace the workspace
static int check_no_pending(const kge_handle *h, const char *fn)
{
    if (h->sum_pending)
        return fail(KGE_ERR_INVALID_ARGUMENT, "%s: the replaced-row sum of a deferred step is pending in the training workspace "
                                              "(kge_optimizer_step_deferred first)", fn);
    return KGE_OK;
}

extern "C" int kge_set_train_workspace(kge_handle *h, void *ws_dev, int64_t bytes, void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_set_train_workspace");
    if (bytes < 0 || (ws_dev && ((uintptr_t)ws_dev & 15)))
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_set_train_workspace: bytes < 0 or workspace not 16-byte aligned");
    if (int rc = check_no_pending(h, "kge_set_train_workspace")) return rc;
    Carve counts(nullptr);
    carve_train_workspace(h, 0, counts);
    if (ws_dev && bytes < (int64_t)counts.at)
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_set_train_workspace: %lld bytes do not hold the per-entity counts", (long long)bytes);
    if (ws_dev) KGE_CUDA(cudaMemsetAsync(ws_dev, 0, 4 * (size_t)h->cfg.n_ent, (cudaStream_t)stream), "kge_set_train_workspace");
    h->train_ws = ws_dev;
    h->train_ws_bytes = ws_dev ? bytes : 0;
    return KGE_OK;
}

// NSCaching: refresh the batch's cache rows, then draw the step's corruptions from them (kge_nscaching.cu)
extern "C" int kge_nscaching_step(kge_handle *h, const kge_nscaching *cache, const float *ent_dev, const float *rel_dev,
                                  const int32_t *triples_dev, const int32_t *key_rows_dev, const uint8_t *update_dev,
                                  int64_t B, uint64_t seed, uint64_t step, int32_t *neg_ent_dev,
                                  uint8_t *neg_keep_subj_dev, uint64_t *misses_dev, void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_nscaching_step");
    const kge_nscaching *q = cache;
    if (!q || q->struct_size != (int32_t)sizeof(kge_nscaching))
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_nscaching_step: bad kge_nscaching (ABI mismatch)");
    if (q->cache_size < 1 || q->random_size < 1 || q->cache_size > 512 - q->random_size)
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_nscaching_step: need cache_size >= 1, random_size >= 1 and their sum "
                                              "<= 512, got %d and %d", q->cache_size, q->random_size);
    if (q->sub_n_keys < 1 || q->obj_n_keys < 1 || !q->sub_ids_dev || !q->sub_count_dev || !q->obj_ids_dev || !q->obj_count_dev)
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_nscaching_step: a side without cache rows or with null cache arrays");
    NSCacheParams p;
    memset(&p, 0, sizeof(p));
    if (int rc = side_filters(q, "kge_nscaching_step", p)) return rc;
    if (int rc = check_sampled_batch(h, B, "kge_nscaching_step")) return rc;
    if (B == 0) return KGE_OK;
    if (!ent_dev || !rel_dev || !triples_dev || !key_rows_dev || !update_dev || !neg_ent_dev || !neg_keep_subj_dev)
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_nscaching_step: null table, triples, key rows, flags or output pointer");
    if (int rc = check_no_pending(h, "kge_nscaching_step")) return rc;
    if (int rc = check_no_stash(h, "kge_nscaching_step")) return rc;
    const size_t smem = nscaching_smem_bytes(h->L.ld, q->cache_size, q->random_size);
    if ((long long)smem > h->max_smem)
        return fail(KGE_ERR_UNSUPPORTED, "kge_nscaching_step: rows of %d floats and %d candidates exceed the shared memory "
                                         "of the refresh kernel (%d B)", h->L.ld, q->cache_size + q->random_size, h->max_smem);
    cudaStream_t st = (cudaStream_t)stream;
    if (int rc = refresh_rotation(h, rel_dev, st)) return rc;
    p.ent = ent_dev;
    p.rel = relation_rows(h, rel_dev);
    p.triples = triples_dev;
    p.key_rows = key_rows_dev;
    p.update = update_dev;
    p.B = B;
    p.model = h->cfg.scoring;
    p.kp = h->L.kp;
    p.ld = h->L.ld;
    p.eta = h->cfg.eta;
    p.n1 = q->cache_size;
    p.n2 = q->random_size;
    p.n_ent = (unsigned)h->cfg.n_ent;
    p.scale = h->score_scale;
    p.seed = seed;
    p.step = step;
    p.ids[0] = q->sub_ids_dev;
    p.count[0] = q->sub_count_dev;
    p.ids[1] = q->obj_ids_dev;
    p.count[1] = q->obj_count_dev;
    p.neg_ent = neg_ent_dev;
    p.neg_keep = neg_keep_subj_dev;
    p.misses = reinterpret_cast<unsigned long long *>(misses_dev);
    KGE_CUDA(launch_nscaching(p, h->sm_count, st), "kge_nscaching_step");
    return KGE_OK;
}

// Carve-up of the shared-negatives workspace for B positives: [B, eta] scores, [B] positive scores, [B, eta] sides
static void carve_shared_negatives(const kge_handle *h, int64_t B, Carve &c, SharedNegParams *q)
{
    const size_t n = (size_t)h->cfg.eta * (size_t)B;
    float *sc = c.take<float>(4 * n, 16);
    float *pos = c.take<float>(4 * (size_t)B, 16);
    uint8_t *keep = c.take<uint8_t>(n, 16);
    if (q) { q->sc = sc; q->pos = pos; q->keep = keep; }
}

extern "C" int64_t kge_shared_negatives_workspace_bytes(const kge_handle *h, int64_t B, int64_t chunk)
{
    if (!h || B < 0 || chunk < 1) return 0;
    Carve c(nullptr);
    carve_shared_negatives(h, B, c, nullptr);
    return (int64_t)c.at;
}

// Shared negatives: the score, loss and gradient passes of kge_train_shared.cu
extern "C" int kge_shared_negatives_step(kge_handle *h, int64_t chunk, const float *ent_dev, const float *rel_dev,
                                         float *grad_ent_dev, float *grad_rel_dev, const int32_t *triples_dev, int64_t B,
                                         const kge_negative_sampler *sampler, uint64_t seed, uint64_t step,
                                         double *loss_dev, void *workspace_dev, int64_t ws_bytes, void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_shared_negatives_step");
    if (chunk < 1) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_shared_negatives_step: chunk must be >= 1, got %lld", (long long)chunk);
    if (int rc = check_sampled_batch(h, B, "kge_shared_negatives_step")) return rc;
    const kge_negative_sampler *s = sampler;
    if (s)
        if (int rc = check_sampler(s, "kge_shared_negatives_step")) return rc;
    if (int rc = check_no_pending(h, "kge_shared_negatives_step")) return rc;
    if (s && (s->sub_pool_off_dev || s->sub_pool_ids_dev || s->obj_pool_off_dev || s->obj_pool_ids_dev ||
              s->sub_filter_n != 0 || s->obj_filter_n != 0))
        return fail(KGE_ERR_UNSUPPORTED, "kge_shared_negatives_step: a sampler with pools or a filter picks entities per "
                                         "positive, and shared negatives draw one candidate set per chunk");
    if (int rc = check_no_stash(h, "kge_shared_negatives_step")) return rc;
    if (int rc = check_no_dropout(h, "kge_shared_negatives_step")) return rc;
    if (B == 0) return KGE_OK;
    if (!ent_dev || !rel_dev || !grad_ent_dev || !grad_rel_dev || !triples_dev || !workspace_dev)
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_shared_negatives_step: null table, gradient, triples or workspace pointer");
    const int64_t need = kge_shared_negatives_workspace_bytes(h, B, chunk);
    if (ws_bytes < need || ((uintptr_t)workspace_dev & 15))
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_shared_negatives_step: workspace of %lld bytes (need %lld, 16-byte "
                                              "aligned)", (long long)ws_bytes, (long long)need);
    const long long ctas = shared_negatives_grid(B, chunk, h->cfg.eta, nullptr);
    if (ctas >= (1ll << 31))
        return fail(KGE_ERR_UNSUPPORTED, "kge_shared_negatives_step: %lld CTAs exceed one launch", ctas);
    cudaStream_t st = (cudaStream_t)stream;
    if (int rc = refresh_rotation(h, rel_dev, st)) return rc;
    SharedNegParams q;
    memset(&q, 0, sizeof(q));
    q.t = sampled_train_params(h, ent_dev, rel_dev, grad_ent_dev, grad_rel_dev, triples_dev, B, seed, step, loss_dev);
    q.chunk = chunk;
    q.thr = s ? s->thresholds_dev : nullptr;
    Carve c(workspace_dev);
    carve_shared_negatives(h, B, c, &q);
    shared_negatives_grid(B, chunk, h->cfg.eta, &q);
    KGE_CUDA(launch_shared_negatives(q, h->sm_count, st), "kge_shared_negatives_step");
    return KGE_OK;
}

static int train_step_impl(kge_handle *h, int32_t mode, const kge_shard_map *map, const float *ent_dev,
                           const float *rel_dev, float *grad_ent_dev, float *grad_rel_dev,
                           const int32_t *triples_dev, int64_t B, const int32_t *neg_ent_dev,
                           const uint8_t *neg_keep_subj_dev, uint64_t seed, uint64_t step, double *loss_dev,
                           float *scores_pos_dev, float *scores_neg_dev, const float *dpos_dev,
                           const float *dneg_dev, void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_train_step");
    if (int rc = check_no_dropout(h, map ? "kge_train_step_sharded" : "kge_train_step")) return rc;
    if (mode < KGE_STEP_FUSED || mode > KGE_STEP_FUSED_DEFER)
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_train_step: unknown mode %d", mode);
    if (int rc = check_no_pending(h, "kge_train_step")) return rc;
    const bool defer = mode == KGE_STEP_FUSED_DEFER;
    if (defer) mode = KGE_STEP_FUSED;
    if (B < 0) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_train_step: B < 0");
    if (B == 0) return KGE_OK;
    if (!ent_dev || !rel_dev || !triples_dev) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_train_step: null table/triples");
    if (mode != KGE_STEP_FORWARD_ONLY && (!grad_ent_dev || !grad_rel_dev))
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_train_step: null gradient buffer");
    if ((neg_ent_dev == nullptr) != (neg_keep_subj_dev == nullptr))
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_train_step: neg_ent_dev and neg_keep_subj_dev must be given together");
    if (mode == KGE_STEP_BACKWARD_EXT && (!dpos_dev || !dneg_dev))
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_train_step: BACKWARD_EXT needs dpos_dev and dneg_dev");
    if (mode == KGE_STEP_FORWARD_ONLY && (!scores_pos_dev || !scores_neg_dev))
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_train_step: FORWARD_ONLY needs both score outputs");
    if (h->slot[TRAIN_GENERAL].warps < 1)
        return fail(KGE_ERR_UNSUPPORTED, "kge_train_step: one positive's working set (%d B) exceeds shared memory (%d B)",
                    h->slot[TRAIN_GENERAL].region_bytes, h->max_smem);
    cudaStream_t st = (cudaStream_t)stream;
    if (int rc = refresh_rotation(h, rel_dev, st)) return rc;

    TrainParams p = sampled_train_params(h, ent_dev, rel_dev, grad_ent_dev, grad_rel_dev, triples_dev, B, seed, step,
                                         loss_dev);
    p.mode = mode;
    p.neg_ent = neg_ent_dev;
    p.neg_keep = neg_keep_subj_dev;
    p.scores_pos = scores_pos_dev;
    p.scores_neg = scores_neg_dev;
    p.dpos = dpos_dev;
    p.dneg = dneg_dev;
    p.nbuf = h->nbuf;
    p.wk = h->wk;
    p.n_cb = h->n_cb;
    p.slot_floats = h->slot_floats;
    p.resident = h->resident;
    p.eta_pad = h->eta_pad;
    p.hot_ent[0] = h->hot_ent[0];
    p.hot_ent[1] = h->hot_ent[1];
    p.stash = row_stash(h, B);
    if (map) {
        // the map's stamps replace the handle's for any world (a one-rank map runs the unsharded kernels, which stamp
        // p.stamp_ent directly); all or nothing
        p.stamp_ent = map->stamp_ent[0];
        for (int q = 0; q < map->world; ++q) {
            p.stamp_ent_shard[q] = map->stamp_ent[q];
            if (!map->stamp_ent[q]) p.stamp_ent = nullptr;
        }
    }
    if (map && map->world > 1) {
        p.shard_world = map->world;
        p.rows_per_shard = (int)map->rows_per_shard;
        for (int q = 0; q < map->world; ++q) { p.ent_shard[q] = map->ent[q]; p.grad_ent_shard[q] = map->grad_ent[q]; }
    }
    const TrainPath path = train_path(h, map, p.stash);
    const TrainSlot &slot = h->slot[path];
    p.G = slot.G;
    p.rows_bytes = slot.rows_bytes;
    p.region_bytes = slot.region_bytes;
    // Dynamic assignment of positives to warps (kge_train_common.cuh) where it was measured to pay before the H100 port: the resident fast path on
    // tables that live in L2 with enough positives per warp for the imbalance to matter (cfg2).  On an HBM-resident table it
    // LOSES (and the general kernel on cfg4 / cfg5w gains nothing), so those keep the static stride.  KGE_B200_TRAIN_SCHED=static|dynamic forces.
    {
        const char *ev = getenv("KGE_B200_TRAIN_SCHED");
        const long long n_warps = (long long)h->sm_count * slot.warps;
        bool dyn = path == TRAIN_RES && B >= 8 * n_warps && 2ll * h->cfg.n_ent * h->L.ld * 4 <= (long long)h->l2_bytes;
        if (ev && strcmp(ev, "static") == 0) dyn = false;
        if (ev && strcmp(ev, "dynamic") == 0) dyn = true;
        p.sched = (dyn && B < (1ll << 24)) ? h->done_counter + 1 : nullptr;  // float counter: exact below 2^24
        // The hot-entity privatisation (kge_set_hot_entities) was a remedy for the same imbalance -- warps that drew many
        // positives of a hot entity fell behind on its serialised atomics -- and with the dynamic assignment it only costs
        // time in bench.py's workload.  It stays in effect for the static stride, where it pays.
        if (p.sched) p.hot_ent[0] = p.hot_ent[1] = -1;
    }
    auto defer_unsupported = [&]() {
        return fail(KGE_ERR_UNSUPPORTED, "kge_train_step: KGE_STEP_FUSED_DEFER needs a step that sums the replaced rows per "
                                         "entity (kge_train_workspace_bytes(h, B) > 0 and a workspace that holds it)");
    };
    if (path == TRAIN_ROT) {
        if (defer) return defer_unsupported();
        KGE_CUDA(launch_train_rot(p, h->nit, slot, h->sm_count, st), "kge_train_step");
        return KGE_OK;
    }
    if (path == TRAIN_RES) {
        // Owner-computes gradient of the replaced rows (kge_train_bucket.cu) where it applies and the workspace set holds it
        // (train_ws_bytes is 0 without one): on H100 the eta*B uniformly scattered row REDs it removes cost about half the
        // kernel (DESIGN.md 3.2, 5).
        const int64_t need = mode != KGE_STEP_FORWARD_ONLY ? bucket_workspace_bytes(h, B) : 0;
        const bool gather = need > 0 && need <= h->train_ws_bytes;
        if (defer && !gather) return defer_unsupported();
        if (gather) {
            Carve c(h->train_ws);
            p.bk = carve_train_workspace(h, B, c);
            KGE_CUDA(launch_bucket_prepass(p, st), "kge_train_step (bucket pre-pass)");
        }
        KGE_CUDA(launch_train_res(p, h->nit, slot, h->sm_count, st), "kge_train_step");
        if (defer) {
            h->pending = p;
            h->sum_pending = true;
        } else if (gather) {
            KGE_CUDA(launch_bucket_sum(p, h->nit, st), "kge_train_step (bucket sum)");
        }
        return KGE_OK;
    }
    if (defer) return defer_unsupported();
    KGE_CUDA(launch_train(p, h->nit, slot, h->sm_count, st), "kge_train_step");
    return KGE_OK;
}

extern "C" int kge_train_step(kge_handle *h, int32_t mode, const float *ent_dev, const float *rel_dev,
                              float *grad_ent_dev, float *grad_rel_dev, const int32_t *triples_dev, int64_t B,
                              const int32_t *neg_ent_dev, const uint8_t *neg_keep_subj_dev, uint64_t seed,
                              uint64_t step, double *loss_dev, float *scores_pos_dev, float *scores_neg_dev,
                              const float *dpos_dev, const float *dneg_dev, void *stream)
{
    return train_step_impl(h, mode, nullptr, ent_dev, rel_dev, grad_ent_dev, grad_rel_dev, triples_dev, B, neg_ent_dev,
                           neg_keep_subj_dev, seed, step, loss_dev, scores_pos_dev, scores_neg_dev, dpos_dev, dneg_dev,
                           stream);
}

extern "C" int kge_train_step_sharded(kge_handle *h, int32_t mode, const kge_shard_map *map, const float *rel_dev,
                                      float *grad_rel_dev, const int32_t *triples_dev, int64_t B,
                                      const int32_t *neg_ent_dev, const uint8_t *neg_keep_subj_dev, uint64_t seed,
                                      uint64_t step, double *loss_dev, float *scores_pos_dev,
                                      float *scores_neg_dev, const float *dpos_dev, const float *dneg_dev,
                                      void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_train_step_sharded");
    if (int rc = check_shard_map(h, map, "kge_train_step_sharded")) return rc;
    if (mode != KGE_STEP_FORWARD_ONLY)
        for (int q = 0; q < map->world; ++q)
            if (!map->grad_ent[q]) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_train_step_sharded: null gradient shard pointer for rank %d", q);
    return train_step_impl(h, mode, map, map->ent[0], rel_dev, map->grad_ent[0], grad_rel_dev, triples_dev, B,
                           neg_ent_dev, neg_keep_subj_dev, seed, step, loss_dev, scores_pos_dev, scores_neg_dev,
                           dpos_dev, dneg_dev, stream);
}

// Checks a caller's config, copies it into out, widened to the current layout, and re-points opt at the copy.  A config
// of an older layout -- before rho (struct_size == offsetof(kge_optimizer_config, rho)) or before l1 -- is accepted for
// the kinds that layout knew; its new fields read as 0.
static int check_optim(const kge_optimizer_config *&opt, const char *fn, kge_optimizer_config &out)
{
    const int32_t size_v1 = (int32_t)offsetof(kge_optimizer_config, rho), size_v2 = (int32_t)offsetof(kge_optimizer_config, l1);
    if (!opt || (opt->struct_size != (int32_t)sizeof(kge_optimizer_config) && opt->struct_size != size_v1 &&
                 opt->struct_size != size_v2))
        return fail(KGE_ERR_INVALID_ARGUMENT, "%s: bad kge_optimizer_config (ABI mismatch)", fn);
    const int last = opt->struct_size == size_v1 ? KGE_OPT_ADAGRAD : opt->struct_size == size_v2 ? KGE_OPT_ADAMAX : KGE_OPT_FTRL;
    if (opt->kind < KGE_OPT_SGD || opt->kind > last)
        return fail(KGE_ERR_INVALID_ARGUMENT, "Could not interpret optimizer identifier: %d", opt->kind);
    if (opt->reg_p < 0 || opt->reg_p2 < 0 || (opt->reg_p == 0 && opt->reg_p2 != 0))
        return fail(KGE_ERR_INVALID_ARGUMENT, "%s: bad regulariser (reg_p >= 0; reg_p2 needs reg_p)", fn);
    memset(&out, 0, sizeof(out));
    memcpy(&out, opt, (size_t)opt->struct_size);
    out.struct_size = (int32_t)sizeof(kge_optimizer_config);
    opt = &out;
    if (out.kind == KGE_OPT_RMSPROP && out.centered && out.momentum != 0.f)
        return fail(KGE_ERR_UNSUPPORTED, "%s: centered RMSprop with momentum needs a third slot buffer (not supported)", fn);
    // Keras' legacy Ftrl refuses the same values (and the NaNs these comparisons also refuse)
    if (out.kind == KGE_OPT_FTRL && !(out.lr_power <= 0.f && out.l1 >= 0.f && out.l2 >= 0.f && out.l2_shrinkage >= 0.f))
        return fail(KGE_ERR_INVALID_ARGUMENT, "%s: Ftrl needs lr_power <= 0 and l1, l2, l2_shrinkage >= 0", fn);
    return KGE_OK;
}
static RegParams reg_of(const kge_optimizer_config *opt)
{
    RegParams r;
    r.p = opt->reg_p; r.lambda = opt->reg_lambda; r.p2 = opt->reg_p2; r.lambda2 = opt->reg_lambda2;
    return r;
}
static OptimParams optim_params(const kge_optimizer_config *opt, int64_t t)
{
    OptimParams o;
    o.kind = opt->kind;
    o.lr = opt->learning_rate;
    o.beta1 = opt->beta_1;
    o.beta2 = opt->beta_2;
    o.eps = opt->epsilon;
    o.momentum = opt->momentum;
    o.reg = reg_of(opt);
    o.rho = opt->rho;
    o.centered = opt->centered;
    // the bias-corrected step, in fp64 on the host and rounded once: legacy Adam lr*sqrt(1 - beta2^t)/(1 - beta1^t),
    // Adamax lr/(1 - beta1^t)
    if (opt->kind == KGE_OPT_ADAMAX)
        o.lr_t = (float)((double)opt->learning_rate / (1.0 - pow((double)opt->beta_1, (double)t)));
    else
        o.lr_t = (float)((double)opt->learning_rate * sqrt(1.0 - pow((double)opt->beta_2, (double)t)) /
                         (1.0 - pow((double)opt->beta_1, (double)t)));
    return o;
}
// Nadam's and Ftrl's per-step scalars, in fp32 as Keras forms them (1 - m_t, 1 - s_new, 1 - s_next: _prepare_local;
// Ftrl's l2 + beta / (2 lr): _resource_apply_dense), and no row-decay mode
static OptimStep optim_step(const kge_optimizer_config *opt)
{
    OptimStep q;
    memset(&q, 0, sizeof(q));
    if (opt->kind == KGE_OPT_FTRL) {
        const float l2 = opt->l2 + opt->ftrl_beta / (2.f * opt->learning_rate);
        q.l1 = opt->l1;
        q.l2x2 = 2.f * l2;
        q.shrinkx2 = 2.f * opt->l2_shrinkage;
        q.lr_power = opt->lr_power;
    } else if (opt->kind == KGE_OPT_NADAM) {
        q.one_m_mt = 1.f - opt->nadam_m_t;
        q.m_t1 = opt->nadam_m_t1;
        q.one_m_snew = 1.f - opt->nadam_s_new;
        q.one_m_snext = 1.f - opt->nadam_s_next;
        q.v_den = opt->nadam_v_den;
    }
    return q;
}
// Every slot buffer the config's update reads and writes must be given
static int check_slots(const kge_optimizer_config *opt, const float *s0, const float *s1, const char *fn)
{
    if ((uses_slot0(opt->kind, opt->momentum) && !s0) || (uses_slot1(opt->kind, opt->momentum, opt->centered) && !s1))
        return fail(KGE_ERR_INVALID_ARGUMENT, "%s: optimizer slot buffer missing", fn);
    return KGE_OK;
}

extern "C" int kge_optimizer_step(kge_handle *h, const kge_optimizer_config *opt, int64_t t, float *table_dev,
                                  float *grad_dev, float *slot0_dev, float *slot1_dev, int64_t rows,
                                  double *reg_loss_dev, void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_optimizer_step");
    kge_optimizer_config cfg;
    if (int rc = check_optim(opt, "kge_optimizer_step", cfg)) return rc;
    if (rows < 0 || t < 1) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_optimizer_step: rows >= 0 and t >= 1 required");
    if (rows == 0) return KGE_OK;
    if (!table_dev || !grad_dev) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_optimizer_step: null table/grad");
    if (int rc = check_slots(opt, slot0_dev, slot1_dev, "kge_optimizer_step")) return rc;
    const OptimParams o = optim_params(opt, t);
    KGE_CUDA(launch_optimizer(o, optim_step(opt), table_dev, grad_dev, slot0_dev, slot1_dev, rows * (long long)h->L.ld, reg_loss_dev,
                              h->sm_count, (cudaStream_t)stream),
             "kge_optimizer_step");
    return KGE_OK;
}

extern "C" int kge_optimizer_step_deferred(kge_handle *h, const kge_optimizer_config *opt, int64_t t, const float *params_in,
                                           float *params_out, float *grad_dev, float *slot0_dev, float *slot1_dev,
                                           int64_t rows, double *reg_loss_dev, void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_optimizer_step_deferred");
    if (!h->sum_pending) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_optimizer_step_deferred: no deferred step is pending");
    kge_optimizer_config cfg;
    if (int rc = check_optim(opt, "kge_optimizer_step_deferred", cfg)) return rc;
    if (t < 1) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_optimizer_step_deferred: t >= 1 required");
    const TrainParams &p = h->pending;
    const size_t ent_floats = (size_t)h->cfg.n_ent * h->L.ld;
    if (rows != h->cfg.n_ent + h->cfg.n_rel || params_in != p.ent || params_in + ent_floats != p.rel ||
        grad_dev != p.grad_ent || grad_dev + ent_floats != p.grad_rel)
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_optimizer_step_deferred: params_in / grad_dev must be the [ent | rel] blocks "
                                              "(n_ent + n_rel rows) the deferred step trained on");
    if (!params_out || params_out == params_in)
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_optimizer_step_deferred: params_out must be a second block");
    if (int rc = check_slots(opt, slot0_dev, slot1_dev, "kge_optimizer_step_deferred")) return rc;
    const OptimParams o = optim_params(opt, t);
    // the checks above refuse without touching the pending step (the caller may repeat the call); from here on it is
    // consumed, and the workspace is free again, whether or not the launch succeeds
    h->sum_pending = false;
    KGE_CUDA(launch_bucket_sum_optimizer(p, h->nit, o, optim_step(opt), params_in, params_out, grad_dev, slot0_dev, slot1_dev, rows,
                                         reg_loss_dev, (cudaStream_t)stream),
             "kge_optimizer_step_deferred");
    return KGE_OK;
}

extern "C" int kge_set_row_stamps(kge_handle *h, int32_t *ent_stamps_dev, int32_t *rel_stamps_dev)
{
    KGE_CHECK_HANDLE(h, "kge_set_row_stamps");
    h->stamp_ent = ent_stamps_dev;
    h->stamp_rel = rel_stamps_dev;
    return KGE_OK;
}

extern "C" int kge_rows_resident(const kge_handle *h) { return h ? (h->resident ? 1 : 0) : -1; }

extern "C" int kge_set_hot_entities(kge_handle *h, const int32_t *ids_host, int32_t n)
{
    KGE_CHECK_HANDLE(h, "kge_set_hot_entities");
    if (n < 0 || (n > 0 && !ids_host)) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_set_hot_entities: bad arguments");
    h->hot_ent[0] = h->hot_ent[1] = -1;
    for (int i = 0; i < n && i < 2; ++i) {
        if (ids_host[i] < 0 || ids_host[i] >= h->cfg.n_ent) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_set_hot_entities: id %d out of range", ids_host[i]);
        if (i == 1 && ids_host[1] == ids_host[0]) break;
        h->hot_ent[i] = ids_host[i];
    }
    return KGE_OK;
}

extern "C" int kge_set_row_stash(kge_handle *h, float *stash_dev, int64_t rows)
{
    KGE_CHECK_HANDLE(h, "kge_set_row_stash");
    if (rows < 0) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_set_row_stash: rows < 0");
    h->stash = stash_dev;
    h->stash_rows = stash_dev ? rows : 0;
    return KGE_OK;
}

extern "C" int32_t kge_step_stamp(uint64_t step) { return (int32_t)(step & 0x3fffffffu) + 1; }

extern "C" int kge_optimizer_step_lazy(kge_handle *h, const kge_optimizer_config *opt, int64_t t, float *table_dev,
                                       float *grad_dev, float *slot0_dev, float *slot1_dev, int64_t rows,
                                       const int32_t *row_stamp_dev, int32_t stamp, double *reg_loss_dev, void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_optimizer_step_lazy");
    kge_optimizer_config cfg;
    if (int rc = check_optim(opt, "kge_optimizer_step_lazy", cfg)) return rc;
    if (rows < 0 || t < 1) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_optimizer_step_lazy: rows >= 0 and t >= 1 required");
    if (rows == 0) return KGE_OK;
    if (!table_dev || !grad_dev || !row_stamp_dev) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_optimizer_step_lazy: null pointer");
    if (int rc = check_slots(opt, slot0_dev, slot1_dev, "kge_optimizer_step_lazy")) return rc;
    const OptimParams o = optim_params(opt, t);
    KGE_CUDA(launch_optimizer_lazy(o, optim_step(opt), table_dev, grad_dev, slot0_dev, slot1_dev, rows, h->L.ld, (const int *)row_stamp_dev,
                                   stamp, reg_loss_dev, h->sm_count, (cudaStream_t)stream),
             "kge_optimizer_step_lazy");
    return KGE_OK;
}

extern "C" int kge_optimizer_step_decay(kge_handle *h, const kge_optimizer_config *opt, int64_t t, float *table_dev,
                                        float *grad_dev, float *slot0_dev, float *slot1_dev, int64_t rows,
                                        const int32_t *row_stamp_dev, int32_t stamp, void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_optimizer_step_decay");
    kge_optimizer_config cfg;
    if (int rc = check_optim(opt, "kge_optimizer_step_decay", cfg)) return rc;
    if (opt->kind != KGE_OPT_NADAM)
        return fail(KGE_ERR_UNSUPPORTED, "kge_optimizer_step_decay: only Nadam has a row-decay rule");
    if (opt->reg_p != 0)
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_optimizer_step_decay: a regularised table's gradient is dense "
                                              "(kge_optimizer_step)");
    if (rows < 0 || t < 1) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_optimizer_step_decay: rows >= 0 and t >= 1 required");
    if (rows == 0) return KGE_OK;
    if (!table_dev || !grad_dev || !row_stamp_dev) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_optimizer_step_decay: null pointer");
    if (int rc = check_slots(opt, slot0_dev, slot1_dev, "kge_optimizer_step_decay")) return rc;
    OptimStep q = optim_step(opt);
    q.row_stamp = (const int *)row_stamp_dev;
    q.stamp = stamp;
    q.ld4 = h->L.ld / 4;
    KGE_CUDA(launch_optimizer(optim_params(opt, t), q, table_dev, grad_dev, slot0_dev, slot1_dev, rows * (long long)h->L.ld,
                              nullptr, h->sm_count, (cudaStream_t)stream),
             "kge_optimizer_step_decay");
    return KGE_OK;
}

static int check_world(int32_t world, int32_t rank, const char *fn)
{
    if (world < 1 || world > KGE_MAX_PEERS || rank < 0 || rank >= world)
        return fail(KGE_ERR_INVALID_ARGUMENT, "%s: world must be 1..%d and 0 <= rank < world", fn, KGE_MAX_PEERS);
    return KGE_OK;
}

extern "C" int kge_optimizer_step_sharded(kge_handle *h, const kge_optimizer_config *opt, int64_t t, int32_t world,
                                          int32_t rank, float *const *peer_tables, float *const *peer_grads,
                                          float *slot0_shard_dev, float *slot1_shard_dev, int64_t row_begin,
                                          int64_t row_end, double *reg_loss_dev, void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_optimizer_step_sharded");
    kge_optimizer_config cfg;
    if (int rc = check_optim(opt, "kge_optimizer_step_sharded", cfg)) return rc;
    if (int rc = check_world(world, rank, "kge_optimizer_step_sharded")) return rc;
    if (row_begin < 0 || row_end < row_begin || t < 1) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_optimizer_step_sharded: bad row range / t");
    if (row_end == row_begin) return KGE_OK;
    if (!peer_tables || !peer_grads) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_optimizer_step_sharded: null pointer arrays");
    for (int q = 0; q < world; ++q)
        if (!peer_tables[q] || !peer_grads[q]) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_optimizer_step_sharded: null peer pointer for rank %d", q);
    if (int rc = check_slots(opt, slot0_shard_dev, slot1_shard_dev, "kge_optimizer_step_sharded")) return rc;
    const OptimParams o = optim_params(opt, t);
    KGE_CUDA(launch_optimizer_sharded(o, optim_step(opt), world, rank, peer_tables, peer_grads, slot0_shard_dev, slot1_shard_dev,
                                      row_begin * (long long)h->L.ld, (row_end - row_begin) * (long long)h->L.ld,
                                      reg_loss_dev, h->sm_count, (cudaStream_t)stream),
             "kge_optimizer_step_sharded");
    return KGE_OK;
}

extern "C" int kge_optimizer_step_exchange(kge_handle *h, const kge_optimizer_config *opt_ent,
                                           const kge_optimizer_config *opt_rel, int64_t t, int32_t world, int32_t rank,
                                           float *const *peer_tables, float *const *peer_grads, float *table_mc_dev,
                                           const float *grads_mc_dev, float *zero_grads_dev,
                                           float *slot0_shard_dev, float *slot1_shard_dev, int64_t row_begin,
                                           int64_t row_end, uint32_t *const *peer_flags, uint32_t token, int32_t phases,
                                           double *reg_loss_dev, void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_optimizer_step_exchange");
    kge_optimizer_config cfg_ent, cfg_rel;
    if (int rc = check_optim(opt_ent, "kge_optimizer_step_exchange", cfg_ent)) return rc;
    if (int rc = check_optim(opt_rel, "kge_optimizer_step_exchange", cfg_rel)) return rc;
    if (int rc = check_world(world, rank, "kge_optimizer_step_exchange")) return rc;
    if (opt_ent->kind != opt_rel->kind || opt_ent->learning_rate != opt_rel->learning_rate || opt_ent->beta_1 != opt_rel->beta_1 ||
        opt_ent->beta_2 != opt_rel->beta_2 || opt_ent->epsilon != opt_rel->epsilon || opt_ent->momentum != opt_rel->momentum ||
        opt_ent->rho != opt_rel->rho || opt_ent->centered != opt_rel->centered ||
        memcmp(&opt_ent->l1, &opt_rel->l1, sizeof(kge_optimizer_config) - offsetof(kge_optimizer_config, l1)) != 0)
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_optimizer_step_exchange: the two tables may differ in their regulariser only");
    const int64_t total_rows = h->cfg.n_ent + h->cfg.n_rel;
    if (row_begin < 0 || row_end < row_begin || row_end > total_rows || t < 1)
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_optimizer_step_exchange: bad row range / t");
    if (phases < 0 || phases > 3) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_optimizer_step_exchange: phases must be 0..3");
    if (!peer_tables || !peer_grads || (phases && !peer_flags))
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_optimizer_step_exchange: null pointer arrays");
    for (int q = 0; q < world; ++q)
        if (!peer_tables[q] || !peer_grads[q] || (phases && !peer_flags[q]))
            return fail(KGE_ERR_INVALID_ARGUMENT, "kge_optimizer_step_exchange: null peer pointer for rank %d", q);
    if (row_end > row_begin)
        if (int rc = check_slots(opt_ent, slot0_shard_dev, slot1_shard_dev, "kge_optimizer_step_exchange")) return rc;
    const OptimParams o = optim_params(opt_ent, t);
    ExchangeParams x;
    memset(&x, 0, sizeof(x));
    x.world = world; x.rank = rank; x.phases = phases;
    for (int q = 0; q < world; ++q) { x.table[q] = peer_tables[q]; x.grad[q] = peer_grads[q]; x.flags[q] = phases ? peer_flags[q] : nullptr; }
    if ((table_mc_dev == nullptr) != (grads_mc_dev == nullptr))
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_optimizer_step_exchange: give both multicast mappings or neither");
    x.table_mc = table_mc_dev;
    x.grad_mc = grads_mc_dev;
    x.token = token;
    x.zero_grad = zero_grads_dev;
    const long long ld4 = h->L.ld / 4;
    x.total4 = total_rows * ld4;
    x.off4 = row_begin * ld4;
    x.n4 = (row_end - row_begin) * ld4;
    x.ent4 = h->cfg.n_ent * ld4;
    x.reg_ent = reg_of(opt_ent);
    x.reg_rel = reg_of(opt_rel);
    x.slot0 = slot0_shard_dev; x.slot1 = slot1_shard_dev;
    x.reg_loss = reg_loss_dev;
    x.done_counter = h->done_counter;
    x.trace = h->exchange_trace;
    KGE_CUDA(launch_optimizer_exchange(o, optim_step(opt_ent), x, h->sm_count, (cudaStream_t)stream), "kge_optimizer_step_exchange");
    return KGE_OK;
}

extern "C" int kge_set_exchange_trace(kge_handle *h, uint64_t *stamps_dev)
{
    KGE_CHECK_HANDLE(h, "kge_set_exchange_trace");
    h->exchange_trace = reinterpret_cast<unsigned long long *>(stamps_dev);
    return KGE_OK;
}

extern "C" int kge_peer_barrier(kge_handle *h, int32_t world, int32_t rank, uint32_t *const *peer_flags, int32_t slot,
                                uint32_t token, void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_peer_barrier");
    if (int rc = check_world(world, rank, "kge_peer_barrier")) return rc;
    if (slot < 0 || slot > 1 || !peer_flags) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_peer_barrier: bad slot / null flags");
    for (int q = 0; q < world; ++q)
        if (!peer_flags[q]) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_peer_barrier: null flag pad for rank %d", q);
    KGE_CUDA(launch_peer_barrier(world, rank, peer_flags, slot, token, (cudaStream_t)stream), "kge_peer_barrier");
    return KGE_OK;
}

// ---- ranking ---------------------------------------------------------------------------------------------
// caller-owned workspace, carved into 256-byte aligned regions
struct RankWorkspace {
    float *qs, *qo, *qaux;   // [b, ld] query vectors (subject side / object side / RotatE object rows)
    int32_t *qpos, *cnt;     // [b], [b,3]
    bool tc;                 // tensor-core filter region present (KGE_RANK_MODE_AUTO, bilinear model, large enough call)
    RankTcLayout tcl;
    void *tc_base;
};
// tc_region = false: never carve the tensor-core region (kge_topk runs the exact chain only)
static RankWorkspace carve_rank_workspace(const kge_handle *h, Carve &c, int64_t b, int64_t n_cand, bool tc_region)
{
    RankWorkspace w;
    const size_t qbytes = (size_t)b * h->L.ld * sizeof(float);
    w.qs = c.take<float>(qbytes, 256);
    w.qo = c.take<float>(qbytes, 256);
    w.qaux = c.take<float>(qbytes, 256);
    w.qpos = c.take<int32_t>((size_t)b * sizeof(int32_t), 256);
    w.cnt = c.take<int32_t>((size_t)3 * b * sizeof(int32_t), 256);
    w.tc = tc_region && h->cfg.rank_mode == KGE_RANK_MODE_AUTO && rank_tc_applicable(h->L, 0, b, n_cand);
    w.tc_base = nullptr;
    if (w.tc) {
        w.tcl = rank_tc_layout(h->L, b, n_cand, h->cfg.rank_pair_cap);
        w.tc_base = c.take<char>(w.tcl.bytes, 1024);  // a multiple of 1024
    }
    return w;
}

extern "C" int64_t kge_rank_workspace_bytes(const kge_handle *h, int64_t b, int64_t n_cand)
{
    if (!h || b < 0 || n_cand < 0) return 0;
    Carve c(nullptr);
    carve_rank_workspace(h, c, b, n_cand, true);
    return (int64_t)c.at;
}

// A caller-owned workspace of `need` bytes (what the sizing function `sizer` returns), `align`-byte aligned
static int check_workspace(void *ws, int64_t bytes, int64_t need, unsigned align, const char *fn, const char *sizer)
{
    if (!ws || bytes < need)
        return fail(KGE_ERR_INVALID_ARGUMENT, "%s: workspace of %lld bytes needed (%s), got %lld", fn, (long long)need, sizer,
                    (long long)(ws ? bytes : 0));
    if ((uintptr_t)ws % align != 0) return fail(KGE_ERR_INVALID_ARGUMENT, "%s: workspace must be %u-byte aligned", fn, align);
    return KGE_OK;
}

// The candidate window of a call over n_rows rows (named `rows` in the message): explicit ids, or the range
// [cand_begin, cand_begin + n_cand)
static int check_candidates(const char *fn, const int32_t *cand_ids, int64_t cand_begin, int64_t n_cand, int64_t n_rows,
                            const char *rows)
{
    if (cand_ids && cand_begin != 0) return fail(KGE_ERR_INVALID_ARGUMENT, "%s: cand_begin must be 0 with cand_ids_dev", fn);
    if (!cand_ids && cand_begin + n_cand > n_rows)
        return fail(KGE_ERR_INVALID_ARGUMENT, "%s: candidate range [%lld,%lld) exceeds %s %lld", fn, (long long)cand_begin,
                    (long long)(cand_begin + n_cand), rows, (long long)n_rows);
    return KGE_OK;
}

// The candidate window of a ranking / top-k call on `side`: entity rows, or relation rows on KGE_SIDE_P
static int check_side_candidates(const kge_handle *h, const char *fn, int32_t side, const int32_t *cand_ids, int64_t cand_begin,
                                 int64_t n_cand)
{
    if (side == KGE_SIDE_P) return check_candidates(fn, cand_ids, cand_begin, n_cand, h->cfg.n_rel, "n_rel");
    return check_candidates(fn, cand_ids, cand_begin, n_cand, h->cfg.n_ent, "n_ent");
}

// The query side of a ranking call: refresh the rotation table (RotatE), prepare the b triples' query vectors and
// quantised positive scores into w (launch_rank_prepare; entity rows ent, or the shards of map), and set *p to their
// scoring parameters against ent.  The candidate window and the outputs are the caller's; a CUDA error is reported as
// `what`.
static int prepare_queries(kge_handle *h, const kge_shard_map *map, const RankWorkspace &w, int32_t side, int32_t strategy,
                           const float *ent, const float *rel, const int32_t *triples, int64_t b, cudaStream_t st,
                           const char *what, RankParams *p)
{
    if (int rc = refresh_rotation(h, rel, st)) return rc;
    ShardView sv;
    memset(&sv, 0, sizeof(sv));
    if (map && map->world > 1) {
        sv.world = map->world;
        sv.rows_per_shard = (int)map->rows_per_shard;
        for (int q = 0; q < map->world; ++q) sv.ent[q] = map->ent[q];
    }
    KGE_CUDA(launch_rank_prepare(h->L, sv, ent, rel, h->rot, triples, b, h->score_scale, w.qs, w.qo, w.qaux, w.qpos, st), what);
    memset(p, 0, sizeof(*p));
    p->L = h->L;
    p->side = side;
    p->strategy = strategy;
    p->ent = ent;
    p->qvec = side == KGE_SIDE_S ? w.qs : w.qo;
    p->qaux = w.qaux;
    p->qpos = w.qpos;
    p->b = b;
    p->scale = h->score_scale;
    return KGE_OK;
}

static int rank_impl(kge_handle *h, const kge_shard_map *map, int64_t filt_base, int32_t side, int32_t strategy,
                     const float *ent_dev, const float *rel_dev, const int32_t *triples_dev, int64_t b,
                     const int32_t *cand_ids_dev, int64_t cand_begin, int64_t n_cand, const int64_t *filt_off_dev,
                     const int32_t *filt_idx_dev, int64_t n_filt, int32_t *ranks_dev, int32_t *counts_dev,
                     float *scores_dev, void *workspace_dev, int64_t workspace_bytes, void *stream,
                     float *probe_delta_dev = nullptr)
{
    KGE_CHECK_HANDLE(h, "kge_rank");
    if (side != KGE_SIDE_S && side != KGE_SIDE_O && side != KGE_SIDE_P) return fail(KGE_ERR_INVALID_ARGUMENT, "Invalid value for corrupt_side");
    if (strategy < KGE_RANK_WORST || strategy > KGE_RANK_MIDDLE)
        return fail(KGE_ERR_INVALID_ARGUMENT, "Invalid value for ranking_strategy");
    if (b < 0 || n_cand < 0 || cand_begin < 0 || n_filt < 0) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_rank: negative size");
    if (b == 0) return KGE_OK;
    if (!ent_dev || !rel_dev || !triples_dev) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_rank: null pointer");
    if (!ranks_dev && !counts_dev && !scores_dev) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_rank: no output buffer");
    // (a shard's window [0, n_local) always lies inside n_ent)
    if (int rc = check_side_candidates(h, "kge_rank", side, cand_ids_dev, cand_begin, n_cand)) return rc;
    // both filter pointers null with n_filt > 0: nothing is filtered (kge_topk / kge_knn reject that)
    if ((filt_off_dev == nullptr) != (filt_idx_dev == nullptr) && n_filt > 0)
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_rank: filter offsets and indices must be given together");
    if (int rc = check_workspace(workspace_dev, workspace_bytes, kge_rank_workspace_bytes(h, b, n_cand), 1024, "kge_rank",
                                 "kge_rank_workspace_bytes"))
        return rc;
    cudaStream_t st = (cudaStream_t)stream;
    Carve c(workspace_dev);
    const RankWorkspace w = carve_rank_workspace(h, c, b, n_cand, true);
    RankParams p;
    if (int rc = prepare_queries(h, map, w, side, strategy, ent_dev, rel_dev, triples_dev, b, st, "kge_rank: prepare", &p))
        return rc;
    // raw counters of THIS call in a zeroed scratch; added to the caller's accumulator or finalized into ranks_dev below
    int32_t *cnt = w.cnt;
    KGE_CUDA(cudaMemsetAsync(cnt, 0, (size_t)3 * b * sizeof(int32_t), st), "kge_rank: memset");
    p.cand_ids = cand_ids_dev;
    p.cand_begin = cand_begin;
    p.n_cand = n_cand;
    p.filt_base = filt_base;
    p.scores = scores_dev;
    if (probe_delta_dev) {  // kge_rank_filter_probe: approximate scores + assumed bound, nothing is counted
        if (!w.tc || n_cand == 0) return fail(KGE_ERR_UNSUPPORTED, "kge_rank_filter_probe: the tensor-core filter does not apply to this call");
        p.scores = nullptr;
        KGE_CUDA(launch_rank_count_tc(p, w.tcl, w.tc_base, cnt, h->sm_count, st, scores_dev, probe_delta_dev), "kge_rank_filter_probe");
        return KGE_OK;
    }
    if (side == KGE_SIDE_P) {  // relation candidates: the exact chain of every pair in every rank_mode (kge_rank_rel.cu)
        const float *rel_rows = relation_rows(h, rel_dev);
        KGE_CUDA(launch_rank_rel_count(p, rel_rows, triples_dev, cnt, st), "kge_rank: count");
        if (filt_off_dev && n_filt > 0)
            KGE_CUDA(launch_rank_rel_filter(p, rel_rows, triples_dev, (const long long *)filt_off_dev, filt_idx_dev, n_filt, cnt,
                                            h->sm_count, st), "kge_rank: filter");
    } else {
        if (w.tc && !scores_dev && n_cand > 0)  // tensor-core filter + exact refine: bit-identical counters (kge_rank_tc.cu)
            KGE_CUDA(launch_rank_count_tc(p, w.tcl, w.tc_base, cnt, h->sm_count, st), "kge_rank: tensor-core count");
        else
            KGE_CUDA(launch_rank_count(p, cnt, st), "kge_rank: count");
        if (filt_off_dev && n_filt > 0)
            KGE_CUDA(launch_rank_filter_n(p, (const long long *)filt_off_dev, filt_idx_dev, n_filt, cnt, h->sm_count, st), "kge_rank: filter");
    }
    if (counts_dev) KGE_CUDA(launch_rank_accumulate(cnt, b, counts_dev, st), "kge_rank: accumulate");
    else if (ranks_dev) KGE_CUDA(launch_rank_finalize(cnt, b, strategy, ranks_dev, st), "kge_rank: finalize");
    return KGE_OK;
}

extern "C" int kge_rank(kge_handle *h, int32_t side, int32_t strategy, const float *ent_dev, const float *rel_dev,
                        const int32_t *triples_dev, int64_t b, const int32_t *cand_ids_dev, int64_t cand_begin,
                        int64_t n_cand, const int64_t *filt_off_dev, const int32_t *filt_idx_dev, int64_t n_filt,
                        int32_t *ranks_dev, int32_t *counts_dev, void *workspace_dev, int64_t workspace_bytes, void *stream)
{
    return rank_impl(h, nullptr, 0, side, strategy, ent_dev, rel_dev, triples_dev, b, cand_ids_dev, cand_begin, n_cand,
                     filt_off_dev, filt_idx_dev, n_filt, ranks_dev, counts_dev, nullptr, workspace_dev, workspace_bytes, stream);
}

extern "C" int kge_rank_sharded(kge_handle *h, const kge_shard_map *map, int32_t rank, int32_t side, int32_t strategy,
                                const float *rel_dev, const int32_t *triples_dev, int64_t b,
                                const int64_t *filt_off_dev, const int32_t *filt_idx_dev, int64_t n_filt,
                                int32_t *ranks_dev, int32_t *counts_dev, void *workspace_dev, int64_t workspace_bytes,
                                void *stream)
{
    if (side == KGE_SIDE_P)
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_rank_sharded: the relation side is not sharded (the relation table is "
                    "replicated): rank it with kge_rank");
    if (!h) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_rank_sharded: null handle");
    if (int rc = check_shard_map(h, map, "kge_rank_sharded")) return rc;
    if (rank < 0 || rank >= map->world) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_rank_sharded: rank out of range");
    const int64_t first = (int64_t)rank * map->rows_per_shard;
    int64_t n_local = h->cfg.n_ent - first;
    if (n_local > map->rows_per_shard) n_local = map->rows_per_shard;
    if (n_local < 0) n_local = 0;
    return rank_impl(h, map, first, side, strategy, map->ent[rank], rel_dev, triples_dev, b, nullptr, 0, n_local,
                     filt_off_dev, filt_idx_dev, n_filt, ranks_dev, counts_dev, nullptr, workspace_dev, workspace_bytes, stream);
}

extern "C" int kge_rank_finalize(kge_handle *h, const int32_t *counts_dev, int64_t b, int32_t strategy, int32_t *ranks_dev,
                                 void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_rank_finalize");
    if (strategy < KGE_RANK_WORST || strategy > KGE_RANK_MIDDLE)
        return fail(KGE_ERR_INVALID_ARGUMENT, "Invalid value for ranking_strategy");
    if (b < 0) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_rank_finalize: b < 0");
    if (b == 0) return KGE_OK;
    if (!counts_dev || !ranks_dev) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_rank_finalize: null pointer");
    KGE_CUDA(launch_rank_finalize(counts_dev, b, strategy, ranks_dev, (cudaStream_t)stream), "kge_rank_finalize");
    return KGE_OK;
}

extern "C" int kge_corruption_scores(kge_handle *h, int32_t side, const float *ent_dev, const float *rel_dev,
                                     const int32_t *triples_dev, int64_t b, const int32_t *cand_ids_dev,
                                     int64_t cand_begin, int64_t n_cand, float *scores_dev, void *workspace_dev,
                                     int64_t workspace_bytes, void *stream)
{
    if (b > 0 && n_cand > 0 && !scores_dev) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_corruption_scores: null output");
    return rank_impl(h, nullptr, 0, side, KGE_RANK_WORST, ent_dev, rel_dev, triples_dev, b, cand_ids_dev, cand_begin, n_cand,
                     nullptr, nullptr, 0, nullptr, nullptr, scores_dev, workspace_dev, workspace_bytes, stream);
}

extern "C" int kge_rank_filter_probe(kge_handle *h, int32_t side, const float *ent_dev, const float *rel_dev,
                                     const int32_t *triples_dev, int64_t b, const int32_t *cand_ids_dev, int64_t cand_begin,
                                     int64_t n_cand, float *approx_dev, float *delta_dev, void *workspace_dev,
                                     int64_t workspace_bytes, void *stream)
{
    if (!approx_dev || !delta_dev) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_rank_filter_probe: null output");
    if (side == KGE_SIDE_P) return fail(KGE_ERR_UNSUPPORTED, "kge_rank_filter_probe: the tensor-core filter does not apply to the relation side");
    return rank_impl(h, nullptr, 0, side, KGE_RANK_WORST, ent_dev, rel_dev, triples_dev, b, cand_ids_dev, cand_begin, n_cand,
                     nullptr, nullptr, 0, nullptr, nullptr, approx_dev, workspace_dev, workspace_bytes, stream, delta_dev);
}

// ---- top-k link prediction ---------------------------------------------------------------------------------
// the running lists of kge_topk_select_kernel: keys and raw scores [2, b, k] each, state [b]
struct TopkLists {
    unsigned long long *keys;
    float *vals;
    int2 *state;
};
static TopkLists carve_topk_lists(Carve &c, int64_t b, int32_t k)
{
    TopkLists l;
    l.keys = c.take<unsigned long long>((size_t)2 * b * k * sizeof(unsigned long long), 256);
    l.vals = c.take<float>((size_t)2 * b * k * sizeof(float), 256);
    l.state = c.take<int2>((size_t)b * sizeof(int2), 256);
    return l;
}
// Candidates per chunk: the [b, C] fp32 chunk the scoring kernel writes and the select kernel reads back is sized to the
// L2 (50 MB on an H100), so it mostly stays there; multiple of 256 (the scoring tile).  Half the L2 was measured slower
// (DESIGN.md 5): more, smaller scoring launches each end in a partly idle wave.
static int64_t topk_chunk(const kge_handle *h, int64_t b, int64_t n_cand)
{
    int64_t c = h->topk_chunk;
    if (c <= 0) {
        c = (int64_t)h->l2_bytes / (4 * (b > 0 ? b : 1)) / 256 * 256;
        if (c < 256) c = 256;
        if (c < n_cand) {  // equal chunks: no small last chunk whose scoring launch leaves most SMs idle
            const int64_t n_chunks = (n_cand + c - 1) / c;
            c = ((n_cand + n_chunks - 1) / n_chunks + 255) / 256 * 256;
        }
    }
    if (c > n_cand) c = n_cand;
    return c < 1 ? 1 : c;
}
struct TopkWorkspace {
    RankWorkspace r;  // query vectors and the (unused) rank counters of the scoring kernels
    float *chunk;     // [b, C]
    TopkLists l;
};
static TopkWorkspace carve_topk_workspace(const kge_handle *h, Carve &c, int64_t b, int64_t n_cand, int32_t k)
{
    TopkWorkspace w;
    w.r = carve_rank_workspace(h, c, b, n_cand, false);
    w.chunk = c.take<float>((size_t)b * topk_chunk(h, b, n_cand) * sizeof(float), 256);
    w.l = carve_topk_lists(c, b, k);
    return w;
}

extern "C" int64_t kge_topk_workspace_bytes(const kge_handle *h, int64_t b, int64_t n_cand, int32_t k)
{
    if (!h || b < 0 || n_cand < 0 || k < 1) return 0;
    Carve c(nullptr);
    carve_topk_workspace(h, c, b, n_cand, k);
    return (int64_t)c.at;
}

extern "C" int64_t kge_select_topk_workspace_bytes(const kge_handle *h, int64_t b, int64_t n, int32_t k)
{
    if (!h || b < 0 || n < 0 || k < 1) return 0;
    Carve c(nullptr);
    carve_topk_lists(c, b, k);
    return (int64_t)c.at;
}

// The select of b running top-k lists over chunks of scores; with n_filt > 0 the filter pairs exclude the candidate
// positions filt_idx - filt_shift
static TopkSelectParams topk_select_params(const float *scores, int64_t b, int32_t k, const TopkLists &l,
                                           const int64_t *filt_off, const int32_t *filt_idx, int64_t n_filt, int64_t filt_shift)
{
    TopkSelectParams s;
    memset(&s, 0, sizeof(s));
    s.scores = scores;
    s.b = b;
    s.k = k;
    if (n_filt > 0) { s.filt_off = (const long long *)filt_off; s.filt_idx = filt_idx; }
    s.filt_shift = filt_shift;
    s.keys = l.keys;
    s.vals = l.vals;
    s.state = l.state;
    return s;
}
// one chunk of nc columns (row stride nc), the candidate positions c0.., into the running lists
static cudaError_t select_chunk(TopkSelectParams s, int64_t nc, int64_t c0, cudaStream_t st)
{
    s.ld = s.n = nc;
    s.base = c0;
    return launch_topk_select(s, st);
}

static int stage_fail(cudaError_t e, const char *fn, const char *stage)
{
    return fail(KGE_ERR_CUDA, "%s: %s: %s (%s)", fn, stage, cudaGetErrorName(e), cudaGetErrorString(e));
}

// The chunked candidate sweep of kge_topk, kge_knn and the radius calls, over the b queries the caller prepared for p:
// for every chunk of topk_chunk candidates, score them with score(p) into p.scores ([b, nc], row stride nc), then run
// epilogue(nc, c0).  CUDA errors are reported as "<fn>: <stage>".
template <class Score, class Epilogue>
static int sweep(const kge_handle *h, const char *fn, const char *stage, RankParams p, Score score, const int32_t *cand_ids,
                 int64_t cand_begin, int64_t n_cand, cudaStream_t st, Epilogue epilogue)
{
    const int64_t C = topk_chunk(h, p.b, n_cand);
    for (int64_t c0 = 0; c0 < n_cand; c0 += C) {
        const int64_t nc = n_cand - c0 < C ? n_cand - c0 : C;
        p.cand_ids = cand_ids ? cand_ids + c0 : nullptr;
        p.cand_begin = cand_ids ? 0 : cand_begin + c0;
        p.n_cand = nc;
        if (cudaError_t e = score(p)) return stage_fail(e, fn, "scores");
        if (cudaError_t e = epilogue(nc, c0)) return stage_fail(e, fn, stage);
    }
    return KGE_OK;
}

extern "C" int kge_topk(kge_handle *h, int32_t side, const float *ent_dev, const float *rel_dev, const int32_t *triples_dev,
                        int64_t b, const int32_t *cand_ids_dev, int64_t cand_begin, int64_t n_cand,
                        const int64_t *filt_off_dev, const int32_t *filt_idx_dev, int64_t n_filt, int32_t k,
                        int32_t *ids_dev, float *scores_dev, void *workspace_dev, int64_t workspace_bytes, void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_topk");
    if (side != KGE_SIDE_S && side != KGE_SIDE_O && side != KGE_SIDE_P) return fail(KGE_ERR_INVALID_ARGUMENT, "Invalid value for corrupt_side");
    if (k < 1) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_topk: k must be >= 1, got %d", k);
    if (b < 0 || n_cand < 0 || cand_begin < 0 || n_filt < 0) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_topk: negative size");
    if (n_cand > 0x7fffffffLL) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_topk: n_cand must be < 2^31");
    if (b == 0) return KGE_OK;
    if (!ent_dev || !rel_dev || !triples_dev || !ids_dev || !scores_dev) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_topk: null pointer");
    if (int rc = check_side_candidates(h, "kge_topk", side, cand_ids_dev, cand_begin, n_cand)) return rc;
    if ((filt_off_dev == nullptr || filt_idx_dev == nullptr) && n_filt > 0)
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_topk: filter offsets and indices must be given together");
    if (int rc = check_workspace(workspace_dev, workspace_bytes, kge_topk_workspace_bytes(h, b, n_cand, k), 1024, "kge_topk",
                                 "kge_topk_workspace_bytes"))
        return rc;
    cudaStream_t st = (cudaStream_t)stream;
    Carve c(workspace_dev);
    const TopkWorkspace w = carve_topk_workspace(h, c, b, n_cand, k);
    RankParams p;
    if (int rc = prepare_queries(h, nullptr, w.r, side, KGE_RANK_WORST, ent_dev, rel_dev, triples_dev, b, st, "kge_topk: prepare", &p))
        return rc;
    KGE_CUDA(cudaMemsetAsync(w.l.state, 0, (size_t)b * sizeof(int2), st), "kge_topk: memset");
    // the exact FP32 chain in every rank_mode: scores bit-identical to kge_corruption_scores
    p.scores = w.chunk;
    const TopkSelectParams s = topk_select_params(w.chunk, b, k, w.l, filt_off_dev, filt_idx_dev, n_filt, cand_ids_dev ? 0 : cand_begin);
    const float *rel_rows = relation_rows(h, rel_dev);
    auto score = [&](const RankParams &q) {
        return side == KGE_SIDE_P ? launch_rank_rel_count(q, rel_rows, triples_dev, w.r.cnt, st)
                                  : launch_rank_count_op(q, rank_op(h->L.model, side), w.r.cnt, st);
    };
    if (int rc = sweep(h, "kge_topk", "select", p, score, cand_ids_dev, cand_begin, n_cand, st,
                       [&](int64_t nc, int64_t c0) { return select_chunk(s, nc, c0, st); }))
        return rc;
    KGE_CUDA(launch_topk_write(w.l.state, w.l.keys, w.l.vals, b, k, cand_ids_dev, cand_begin, ids_dev, scores_dev, st),
             "kge_topk: write");
    return KGE_OK;
}

extern "C" int kge_select_topk(kge_handle *h, const float *scores_dev, int64_t b, int64_t n, int32_t k, int32_t *pos_dev,
                               float *out_dev, void *workspace_dev, int64_t workspace_bytes, void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_select_topk");
    if (k < 1) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_select_topk: k must be >= 1, got %d", k);
    if (b < 0 || n < 0) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_select_topk: negative size");
    if (n > 0x7fffffffLL) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_select_topk: n must be < 2^31");
    if (b == 0) return KGE_OK;
    if ((n > 0 && !scores_dev) || !pos_dev || !out_dev) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_select_topk: null pointer");
    if (int rc = check_workspace(workspace_dev, workspace_bytes, kge_select_topk_workspace_bytes(h, b, n, k), 1024, "kge_select_topk",
                                 "kge_select_topk_workspace_bytes"))
        return rc;
    cudaStream_t st = (cudaStream_t)stream;
    Carve c(workspace_dev);
    const TopkLists l = carve_topk_lists(c, b, k);
    KGE_CUDA(cudaMemsetAsync(l.state, 0, (size_t)b * sizeof(int2), st), "kge_select_topk: memset");
    KGE_CUDA(select_chunk(topk_select_params(scores_dev, b, k, l, nullptr, nullptr, 0, 0), n, 0, st), "kge_select_topk: select");
    KGE_CUDA(launch_topk_write(l.state, l.keys, l.vals, b, k, nullptr, 0, pos_dev, out_dev, st), "kge_select_topk: write");
    return KGE_OK;
}

// ---- nearest-neighbour and radius search over a point matrix ----------------------------------------------------
// Scratch of kge_knn / kge_radius_neighbors: the gathered query rows, the (unused) rank counters the scoring kernels
// update, one [b, C] chunk of -d (C: the kge_topk rule), then the running lists (kge_knn) or the per-row cursors
// (kge_radius_neighbors).
struct KnnWorkspace {
    float *qvec;     // [b, ld]
    int32_t *cnt;    // [b, 4]: three counters + the zero "positive" of each query
    float *chunk;    // [b, C]
    TopkLists l;     // kge_knn
    long long *cursor;  // [b] kge_radius_neighbors
};
static KnnWorkspace carve_knn_workspace(const kge_handle *h, Carve &c, int64_t b, int64_t n_cand, int32_t k, int32_t ld)
{
    KnnWorkspace w;
    memset(&w, 0, sizeof(w));
    w.qvec = c.take<float>((size_t)b * ld * sizeof(float), 256);
    w.cnt = c.take<int32_t>((size_t)4 * b * sizeof(int32_t), 256);
    w.chunk = c.take<float>((size_t)b * topk_chunk(h, b, n_cand) * sizeof(float), 256);
    if (k > 0) w.l = carve_topk_lists(c, b, k);
    else w.cursor = c.take<long long>((size_t)b * sizeof(long long), 256);
    return w;
}

extern "C" int64_t kge_knn_workspace_bytes(const kge_handle *h, int64_t b, int64_t n_cand, int32_t k, int32_t ld)
{
    if (!h || b < 0 || n_cand < 0 || k < 1 || ld < 4 || ld % 4) return 0;
    Carve c(nullptr);
    carve_knn_workspace(h, c, b, n_cand, k, ld);
    return (int64_t)c.at;
}

extern "C" int64_t kge_radius_workspace_bytes(const kge_handle *h, int64_t b, int64_t n_cand, int32_t ld)
{
    if (!h || b < 0 || n_cand < 0 || ld < 4 || ld % 4) return 0;
    Carve c(nullptr);
    carve_knn_workspace(h, c, b, n_cand, 0, ld);
    return (int64_t)c.at;
}

// the checks kge_knn and kge_radius_neighbors share (b > 0)
static int check_points(const char *fn, int32_t metric, const float *points_dev, int64_t n_points, int32_t ld,
                        const int32_t *query_ids_dev, const int32_t *cand_ids_dev, int64_t cand_begin, int64_t n_cand)
{
    if (metric != KGE_METRIC_EUCLIDEAN && metric != KGE_METRIC_MANHATTAN)
        return fail(KGE_ERR_INVALID_ARGUMENT, "%s: unknown metric %d", fn, metric);
    if (ld < 4 || ld % 4) return fail(KGE_ERR_INVALID_ARGUMENT, "%s: ld must be a positive multiple of 4, got %d", fn, ld);
    if (n_points > 0x7fffffffLL) return fail(KGE_ERR_INVALID_ARGUMENT, "%s: ids are int32 (n_points < 2^31)", fn);
    if (!points_dev || !query_ids_dev) return fail(KGE_ERR_INVALID_ARGUMENT, "%s: null pointer", fn);
    if (((uintptr_t)points_dev & 15u) != 0) return fail(KGE_ERR_INVALID_ARGUMENT, "%s: points_dev must be 16-byte aligned", fn);
    return check_candidates(fn, cand_ids_dev, cand_begin, n_cand, n_points, "n_points");
}

static RankParams knn_rank_params(int32_t ld, const float *points_dev, const KnnWorkspace &w, int64_t b)
{
    RankParams p;
    memset(&p, 0, sizeof(p));
    p.L.model = KGE_TRANSE;  // not read: the op is explicit, and the non-RotatE kernels read only L.ld
    p.L.k = p.L.kp = p.L.ld = p.L.K = ld;
    p.L.halves = 1;
    p.strategy = KGE_RANK_WORST;
    p.ent = points_dev;
    p.qvec = w.qvec;
    p.qpos = w.cnt + 3 * b;
    p.b = b;
    p.scale = 1.f;
    p.scores = w.chunk;
    return p;
}

// The sweep of kge_knn and the radius calls: gather the b query points, then sweep -d (the metric's chain) into w.chunk
template <class Epilogue>
static int point_sweep(const kge_handle *h, const char *fn, const char *stage, int32_t metric, const float *points_dev,
                       int32_t ld, const int32_t *query_ids_dev, int64_t b, const int32_t *cand_ids_dev, int64_t cand_begin,
                       int64_t n_cand, const KnnWorkspace &w, cudaStream_t st, Epilogue epilogue)
{
    if (cudaError_t e = launch_knn_gather(points_dev, ld, query_ids_dev, b, w.qvec, st)) return stage_fail(e, fn, "gather");
    if (cudaError_t e = cudaMemsetAsync(w.cnt, 0, (size_t)4 * b * sizeof(int32_t), st)) return stage_fail(e, fn, "memset");
    const int op = metric == KGE_METRIC_EUCLIDEAN ? OP_L2_SUB : OP_L1_SUB;
    return sweep(h, fn, stage, knn_rank_params(ld, points_dev, w, b),
                 [&](const RankParams &q) { return launch_rank_count_op(q, op, w.cnt, st); }, cand_ids_dev, cand_begin, n_cand,
                 st, epilogue);
}

extern "C" int kge_knn(kge_handle *h, int32_t metric, const float *points_dev, int64_t n_points, int32_t ld,
                       const int32_t *query_ids_dev, int64_t b, const int32_t *cand_ids_dev, int64_t cand_begin, int64_t n_cand,
                       const int64_t *filt_off_dev, const int32_t *filt_idx_dev, int64_t n_filt, int32_t k, int32_t farthest,
                       int32_t *ids_dev, float *dist_dev, void *workspace_dev, int64_t workspace_bytes, void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_knn");
    if (k < 1) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_knn: k must be >= 1, got %d", k);
    if (b < 0 || n_points < 0 || n_cand < 0 || cand_begin < 0 || n_filt < 0) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_knn: negative size");
    if (n_cand > 0x7fffffffLL) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_knn: n_cand must be < 2^31");
    if (b == 0) return KGE_OK;
    if (int rc = check_points("kge_knn", metric, points_dev, n_points, ld, query_ids_dev, cand_ids_dev, cand_begin, n_cand)) return rc;
    if (!ids_dev || !dist_dev) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_knn: null pointer");
    if ((filt_off_dev == nullptr || filt_idx_dev == nullptr) && n_filt > 0)
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_knn: filter offsets and indices must be given together");
    if (int rc = check_workspace(workspace_dev, workspace_bytes, kge_knn_workspace_bytes(h, b, n_cand, k, ld), 1024, "kge_knn",
                                 "kge_knn_workspace_bytes"))
        return rc;
    cudaStream_t st = (cudaStream_t)stream;
    Carve c(workspace_dev);
    const KnnWorkspace w = carve_knn_workspace(h, c, b, n_cand, k, ld);
    KGE_CUDA(cudaMemsetAsync(w.l.state, 0, (size_t)b * sizeof(int2), st), "kge_knn: memset");
    const TopkSelectParams s = topk_select_params(w.chunk, b, k, w.l, filt_off_dev, filt_idx_dev, n_filt, cand_ids_dev ? 0 : cand_begin);
    if (int rc = point_sweep(h, "kge_knn", "select", metric, points_dev, ld, query_ids_dev, b, cand_ids_dev, cand_begin, n_cand, w, st,
                             [&](int64_t nc, int64_t c0) {
                                 if (farthest) {  // +d: the select keeps the largest distances
                                     const cudaError_t e = launch_knn_negate(w.chunk, b * nc, st);
                                     if (e != cudaSuccess) return e;
                                 }
                                 return select_chunk(s, nc, c0, st);
                             }))
        return rc;
    KGE_CUDA(launch_topk_write(w.l.state, w.l.keys, w.l.vals, b, k, cand_ids_dev, cand_begin, ids_dev, dist_dev, st, !farthest),
             "kge_knn: write");
    return KGE_OK;
}

// The checks kge_radius_neighbors, kge_radius_union and kge_radius_min_key share; for b > 0, *w is carved on success
static int check_radius(kge_handle *h, const char *fn, int32_t metric, const float *points_dev, int64_t n_points,
                        int32_t ld, const int32_t *query_ids_dev, int64_t b, const int32_t *cand_ids_dev, int64_t cand_begin,
                        int64_t n_cand, void *workspace_dev, int64_t workspace_bytes, KnnWorkspace *w)
{
    if (b < 0 || n_points < 0 || n_cand < 0 || cand_begin < 0) return fail(KGE_ERR_INVALID_ARGUMENT, "%s: negative size", fn);
    if (n_cand > 0x7fffffffLL) return fail(KGE_ERR_INVALID_ARGUMENT, "%s: n_cand must be < 2^31", fn);
    if (b == 0) return KGE_OK;
    if (int rc = check_points(fn, metric, points_dev, n_points, ld, query_ids_dev, cand_ids_dev, cand_begin, n_cand)) return rc;
    if (int rc = check_workspace(workspace_dev, workspace_bytes, kge_radius_workspace_bytes(h, b, n_cand, ld), 1024, "kge_radius",
                                 "kge_radius_workspace_bytes"))
        return rc;
    Carve c(workspace_dev);
    *w = carve_knn_workspace(h, c, b, n_cand, 0, ld);
    return KGE_OK;
}

extern "C" int kge_radius_neighbors(kge_handle *h, int32_t metric, const float *points_dev, int64_t n_points, int32_t ld,
                                    const int32_t *query_ids_dev, int64_t b, const int32_t *cand_ids_dev, int64_t cand_begin,
                                    int64_t n_cand, float radius, int64_t *offsets_dev, int32_t *nbr_dev,
                                    void *workspace_dev, int64_t workspace_bytes, void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_radius_neighbors");
    KnnWorkspace w;
    if (int rc = check_radius(h, "kge_radius_neighbors", metric, points_dev, n_points, ld, query_ids_dev, b, cand_ids_dev,
                              cand_begin, n_cand, workspace_dev, workspace_bytes, &w))
        return rc;
    if (b == 0) return KGE_OK;
    if (!offsets_dev) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_radius_neighbors: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    KGE_CUDA(cudaMemsetAsync(w.cursor, 0, (size_t)b * sizeof(long long), st), "kge_radius_neighbors: memset");
    const long long *off = nbr_dev ? (const long long *)offsets_dev : nullptr;
    if (int rc = point_sweep(h, "kge_radius_neighbors", nbr_dev ? "emit" : "count", metric, points_dev, ld, query_ids_dev, b,
                             cand_ids_dev, cand_begin, n_cand, w, st, [&](int64_t nc, int64_t c0) {
                                 return launch_radius_chunk(w.chunk, nc, nc, c0, b, radius, cand_ids_dev, cand_begin,
                                                            w.cursor, off, nbr_dev, st);
                             }))
        return rc;
    if (!nbr_dev) KGE_CUDA(launch_radius_counts(w.cursor, b, (long long *)offsets_dev, st), "kge_radius_neighbors: counts");
    return KGE_OK;
}

extern "C" int kge_radius_union(kge_handle *h, int32_t metric, const float *points_dev, int64_t n_points, int32_t ld,
                                const int32_t *query_ids_dev, int64_t b, const int32_t *cand_ids_dev, int64_t cand_begin,
                                int64_t n_cand, float radius, int32_t *parent_dev, void *workspace_dev,
                                int64_t workspace_bytes, void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_radius_union");
    KnnWorkspace w;
    if (int rc = check_radius(h, "kge_radius_union", metric, points_dev, n_points, ld, query_ids_dev, b, cand_ids_dev,
                              cand_begin, n_cand, workspace_dev, workspace_bytes, &w))
        return rc;
    if (b == 0) return KGE_OK;
    if (!parent_dev) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_radius_union: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    return point_sweep(h, "kge_radius_union", "union", metric, points_dev, ld, query_ids_dev, b, cand_ids_dev, cand_begin,
                       n_cand, w, st, [&](int64_t nc, int64_t c0) {
                           return launch_radius_union_chunk(w.chunk, nc, nc, c0, b, radius, query_ids_dev, cand_ids_dev,
                                                            cand_begin, parent_dev, st);
                       });
}

extern "C" int kge_radius_min_key(kge_handle *h, int32_t metric, const float *points_dev, int64_t n_points, int32_t ld,
                                  const int32_t *query_ids_dev, int64_t b, const int32_t *cand_ids_dev, int64_t cand_begin,
                                  int64_t n_cand, float radius, const int32_t *key_dev, int32_t *out_dev,
                                  void *workspace_dev, int64_t workspace_bytes, void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_radius_min_key");
    KnnWorkspace w;
    if (int rc = check_radius(h, "kge_radius_min_key", metric, points_dev, n_points, ld, query_ids_dev, b, cand_ids_dev,
                              cand_begin, n_cand, workspace_dev, workspace_bytes, &w))
        return rc;
    if (b == 0) return KGE_OK;
    if (!key_dev || !out_dev) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_radius_min_key: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    KGE_CUDA(launch_min_key_init(out_dev, b, st), "kge_radius_min_key: init");
    return point_sweep(h, "kge_radius_min_key", "min", metric, points_dev, ld, query_ids_dev, b, cand_ids_dev, cand_begin,
                       n_cand, w, st, [&](int64_t nc, int64_t c0) {
                           return launch_radius_min_key_chunk(w.chunk, nc, nc, c0, b, radius, cand_ids_dev, cand_begin,
                                                              key_dev, out_dev, st);
                       });
}

extern "C" int kge_forest_flatten(kge_handle *h, int32_t *parent_dev, int64_t n, void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_forest_flatten");
    if (n < 0 || n > 0x7fffffffLL) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_forest_flatten: n must be in [0, 2^31)");
    if (n > 0 && !parent_dev) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_forest_flatten: null pointer");
    KGE_CUDA(launch_forest_flatten(parent_dev, n, (cudaStream_t)stream), "kge_forest_flatten");
    return KGE_OK;
}

extern "C" int64_t kge_graph_workspace_bytes(int64_t n_nodes)
{
    if (n_nodes < 0 || n_nodes > 0x7fffffffLL) return 0;
    return (int64_t)graph_workspace_bytes(n_nodes);
}

extern "C" int kge_graph_counts(const int64_t *offsets_dev, const int32_t *nbr_dev, const int32_t *order_dev,
                                int64_t n_nodes, int64_t *tri2_dev, int64_t *sq_dev, int64_t *pot_dev,
                                void *workspace_dev, int64_t workspace_bytes, void *stream)
{
    if (n_nodes < 0 || n_nodes > 0x7fffffffLL)
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_graph_counts: n_nodes must be in [0, 2^31)");
    if (n_nodes == 0) return KGE_OK;
    if (!offsets_dev || !nbr_dev || !order_dev || !tri2_dev || !sq_dev || !pot_dev)
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_graph_counts: null pointer");
    const int64_t need = kge_graph_workspace_bytes(n_nodes);
    if (need == 0) return fail(KGE_ERR_CUDA, "kge_graph_counts: device query failed");
    if (!workspace_dev || workspace_bytes < need)
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_graph_counts: workspace of %lld bytes, need %lld",
                    (long long)workspace_bytes, (long long)need);
    if ((uintptr_t)workspace_dev % 8) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_graph_counts: workspace not 8-byte aligned");
    KGE_CUDA(launch_graph_counts((const long long *)offsets_dev, nbr_dev, order_dev, n_nodes, workspace_dev,
                                 (long long *)tri2_dev, (long long *)sq_dev, (long long *)pot_dev, (cudaStream_t)stream),
             "kge_graph_counts");
    return KGE_OK;
}

// ---- all-candidate training: 1vsAll, relation prediction and KvsAll (kge_train_1vsall.cu) ---------------------------

// What sets the three all-candidate steps apart on the host
struct CandidateRule {
    const char *fn, *training, *sizer;  // entry point, what it trains, its workspace sizing function (messages)
    const char *inputs;                 // its pointer arguments (message of the null-pointer refusal)
    bool relation;    // the candidates are the relation rows (side p, queries Qp), else the entity rows (sides s, o)
    bool multiclass;  // multiclass NLL (row statistics), else KvsAll's element-wise multi-label loss (label masks)
};
static const CandidateRule ONE_VS_ALL = {"kge_one_vs_all_step", "1vsAll", "kge_one_vs_all_workspace_bytes",
                                         "table, gradient or triples", false, true};
static const CandidateRule RELATION_PREDICTION = {"kge_one_vs_all_relation_step", "relation prediction",
                                                  "kge_one_vs_all_relation_workspace_bytes", "table, gradient or triples",
                                                  true, true};
static const CandidateRule K_VS_ALL = {"kge_k_vs_all_step", "KvsAll", "kge_k_vs_all_workspace_bytes",
                                       "table, gradient, queries or labels", false, false};

// The query vectors of a step: the entity sides' (and the quantised positive scores launch_rank_prepare also writes),
// or the relation step's Qp in qs
struct CandidateQueries {
    float *qs, *qo;
    int32_t *qpos;
    SideDropout drop;  // drop.cand / drop.grad_cand: the dropout regions while dropout is set, else nullptr
};

// Carve-up of the workspace of a step of s.B queries into the query vectors and the scratch of s's passes: the row
// statistics of the multiclass loss, the per-split partial Gq rows and, when dX is split over the query tiles, its
// [xsplit, n_cand, ld] partial candidate rows.  Sets s.nsplit and s.xsplit; regions a step does not hold stay nullptr.
static CandidateQueries carve_candidates(const kge_handle *h, const CandidateRule &r, Carve &c, OneVsAllSide &s)
{
    CandidateQueries q = {};
    s.nsplit = one_vs_all_splits(s.B, s.n_cand);
    // dX of the relation step: the same split rule with the roles swapped, query tiles per relation tile
    s.xsplit = r.relation ? one_vs_all_splits(s.n_cand, s.B) : 1;
    const size_t rows = (size_t)s.B * h->L.ld * sizeof(float), col = (size_t)s.B * sizeof(float), ns = (size_t)s.nsplit;
    q.qs = c.take<float>(rows, 16);
    if (!r.relation) {
        q.qo = c.take<float>(rows, 16);
        q.qpos = c.take<int32_t>(col, 16);
    }
    if (r.multiclass) {
        s.pm = c.take<float>(ns * col, 16);
        s.pz = c.take<float>(ns * col, 16);
        s.lt = c.take<float>(col, 16);
        s.row_m = c.take<float>(col, 16);
        s.row_inv = c.take<float>(col, 16);
    }
    s.pgq = c.take<float>(ns * rows, 16);
    if (s.xsplit > 1) s.pgx = c.take<float>((size_t)s.xsplit * s.n_cand * h->L.ld * sizeof(float), 16);
    if (dropout_set(h)) {  // one side at a time: its dropped candidate table and their gradient (kge_dropout.cu)
        const size_t table = (size_t)s.n_cand * h->L.ld * sizeof(float);
        q.drop.cand = c.take<float>(table, 16);
        q.drop.grad_cand = c.take<float>(table, 16);
    }
    return q;
}

// The OneVsAllSide fields every all-candidate step shares; side, col and q are the entry point's, the workspace regions
// carve_candidates' and w start_candidate_step's.  The stamps are written only while the entity buffer is set, like kge_train_step:
// start_candidate_step stamps the candidate rows, the chain pass the batch's other rows (its relation rows; on the
// relation step its s and o rows).
static OneVsAllSide candidate_side(const kge_handle *h, const CandidateRule &r, const float *ent, const float *rel,
                                   float *grad_ent, float *grad_rel, const int32_t *triples, int64_t B, uint64_t step,
                                   double *loss)
{
    OneVsAllSide s;
    memset(&s, 0, sizeof(s));
    s.ent = ent;
    s.rel = rel;
    s.grad_ent = grad_ent;
    s.grad_rel = grad_rel;
    s.cand = r.relation ? rel : ent;
    s.grad_cand = r.relation ? grad_rel : grad_ent;
    s.triples = triples;
    s.B = B;
    s.n_cand = r.relation ? h->cfg.n_rel : h->cfg.n_ent;
    s.kp = h->L.kp;
    s.ld = h->L.ld;
    s.scale = h->score_scale;
    s.weight = 1.f;
    s.loss = loss;
    s.stamp = kge_step_stamp(step);
    s.stamp_ent = h->stamp_ent;
    s.stamp_rel = h->stamp_ent ? h->stamp_rel : nullptr;
    return s;
}

static int64_t candidate_workspace_bytes(const kge_handle *h, const CandidateRule &r, int64_t B)
{
    if (!h || B < 0) return 0;
    OneVsAllSide s = candidate_side(h, r, nullptr, nullptr, nullptr, nullptr, nullptr, B, 0, nullptr);
    Carve c(nullptr);
    carve_candidates(h, r, c, s);
    return (int64_t)c.at;
}

// The refusals of an all-candidate step s, in this order, every one before the first launch: the model; the entry
// point's own arguments (own(): KGE_OK or the code of the refusal it reported) and the reduction; a pending deferred
// step; fewer than two candidates; rows too wide for the kernels' shared-memory tiles; B < 0.  An empty batch passes
// before the pointers and the workspace are checked: the caller returns KGE_OK without launching.  Then null tables,
// gradients or triples (own_null: the entry point's other pointers), and the workspace (16-byte aligned).
template <class Own>
static int check_candidate_step(const kge_handle *h, const CandidateRule &r, const OneVsAllSide &s, int32_t reduction,
                                Own own, bool own_null, void *ws, int64_t ws_bytes)
{
    const int model = h->cfg.scoring;
    if (model != KGE_DISTMULT && model != KGE_COMPLEX && model != KGE_HOLE)
        return fail(KGE_ERR_UNSUPPORTED, "%s: %s training is implemented for DistMult, ComplEx and HolE (inner-product "
                                         "scores); not for scoring type %d", r.fn, r.training, model);
    if (int rc = own()) return rc;
    if (reduction != KGE_REDUCE_SUM && reduction != KGE_REDUCE_MEAN)
        return fail(KGE_ERR_INVALID_ARGUMENT, "Invalid value for reduction!");
    if (int rc = check_no_pending(h, r.fn)) return rc;
    if (s.n_cand < 2) return fail(KGE_ERR_INVALID_ARGUMENT, "%s: needs %s >= 2", r.fn, r.relation ? "n_rel" : "n_ent");
    if ((long long)(r.multiclass ? one_vs_all_smem_bytes(s.ld) : k_vs_all_smem_bytes(s.ld)) > h->max_smem)
        return fail(KGE_ERR_UNSUPPORTED, "%s: rows of %d floats exceed the shared-memory tiles of the %s kernels (%d B)",
                    r.fn, s.ld, r.training, h->max_smem);
    if (s.B < 0) return fail(KGE_ERR_INVALID_ARGUMENT, "%s: B < 0", r.fn);
    if (s.B == 0) return KGE_OK;
    if (!s.ent || !s.rel || !s.grad_ent || !s.grad_rel || !s.triples || own_null)
        return fail(KGE_ERR_INVALID_ARGUMENT, "%s: null %s", r.fn, r.inputs);
    return check_workspace(ws, ws_bytes, candidate_workspace_bytes(h, r, s.B), 16, r.fn, r.sizer);
}

// What every checked all-candidate step does before its passes: set the loss weight of the reduction, carve the
// workspace ws into s and *q, write the entity sides' query vectors, and stamp every candidate row as looked up
static int start_candidate_step(const kge_handle *h, const CandidateRule &r, int32_t reduction, void *ws, uint64_t step,
                                cudaStream_t st, OneVsAllSide &s, CandidateQueries *q)
{
    // mean: a negative's exp weighs 1 / (n_cand - 1) in the multiclass loss, every element 1 / n_ent in KvsAll's
    s.w = reduction == KGE_REDUCE_MEAN ? (float)(1.0 / (double)(r.multiclass ? s.n_cand - 1 : s.n_cand)) : 1.f;
    Carve c(ws);
    *q = carve_candidates(h, r, c, s);
    if (dropout_set(h)) {  // launch_dropout_prepare forms each side's queries from its dropped rows
        // keep iff (word >> 8) >= round(p 2^24); scale = fp32(1 / (1 - p))
        q->drop.seed = h->drop_seed;
        q->drop.step = step;
        q->drop.t_ent = (uint32_t)llround((double)h->drop_p_ent * 16777216.0);
        q->drop.t_rel = (uint32_t)llround((double)h->drop_p_rel * 16777216.0);
        q->drop.scale_ent = (float)(1.0 / (1.0 - (double)h->drop_p_ent));
        q->drop.scale_rel = (float)(1.0 / (1.0 - (double)h->drop_p_rel));
    } else if (!r.relation) {
        ShardView sv;
        memset(&sv, 0, sizeof(sv));
        KGE_CUDA(launch_rank_prepare(h->L, sv, s.ent, s.rel, nullptr, s.triples, s.B, h->score_scale, q->qs, q->qo, nullptr,
                                     q->qpos, st),
                 r.fn);
    }
    if (h->stamp_ent)
        KGE_CUDA(launch_one_vs_all_stamps(r.relation ? h->stamp_rel : h->stamp_ent, s.n_cand, s.stamp, st), r.fn);
    return KGE_OK;
}

extern "C" int64_t kge_one_vs_all_workspace_bytes(const kge_handle *h, int64_t B)
{
    return candidate_workspace_bytes(h, ONE_VS_ALL, B);
}

extern "C" int kge_one_vs_all_step(kge_handle *h, int32_t sides, int32_t loss_reduction, const float *ent_dev,
                                   const float *rel_dev, float *grad_ent_dev, float *grad_rel_dev,
                                   const int32_t *triples_dev, int64_t B, uint64_t step, double *loss_dev, void *ws_dev,
                                   int64_t ws_bytes, void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_one_vs_all_step");
    OneVsAllSide s = candidate_side(h, ONE_VS_ALL, ent_dev, rel_dev, grad_ent_dev, grad_rel_dev, triples_dev,
                                    B, step, loss_dev);
    if (int rc = check_candidate_step(h, ONE_VS_ALL, s, loss_reduction, [&]() -> int {
            if (sides < KGE_ONE_VS_ALL_S || sides > (KGE_ONE_VS_ALL_S | KGE_ONE_VS_ALL_O))
                return fail(KGE_ERR_INVALID_ARGUMENT, "kge_one_vs_all_step: sides must be a non-empty set of "
                                                      "KGE_ONE_VS_ALL_S | KGE_ONE_VS_ALL_O, got %d", sides);
            return KGE_OK;
        }, false, ws_dev, ws_bytes))
        return rc;
    if (B == 0) return KGE_OK;
    cudaStream_t st = (cudaStream_t)stream;
    CandidateQueries q;
    if (int rc = start_candidate_step(h, ONE_VS_ALL, loss_reduction, ws_dev, step, st, s, &q)) return rc;
    for (int side = KGE_SIDE_S; side <= KGE_SIDE_O; ++side) {
        if (!(sides & (side == KGE_SIDE_S ? KGE_ONE_VS_ALL_S : KGE_ONE_VS_ALL_O))) continue;
        s.side = side;
        s.col = side == KGE_SIDE_S ? 0 : 2;
        s.q = side == KGE_SIDE_S ? q.qs : q.qo;
        KGE_CUDA(launch_one_vs_all_side(s, h->L.halves, st, q.drop.cand ? &q.drop : nullptr), "kge_one_vs_all_step");
    }
    return KGE_OK;
}

extern "C" int64_t kge_one_vs_all_relation_workspace_bytes(const kge_handle *h, int64_t B)
{
    return candidate_workspace_bytes(h, RELATION_PREDICTION, B);
}

extern "C" int kge_one_vs_all_relation_step(kge_handle *h, float weight, int32_t loss_reduction, const float *ent_dev,
                                            const float *rel_dev, float *grad_ent_dev, float *grad_rel_dev,
                                            const int32_t *triples_dev, int64_t B, uint64_t step, double *loss_dev,
                                            void *ws_dev, int64_t ws_bytes, void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_one_vs_all_relation_step");
    OneVsAllSide s = candidate_side(h, RELATION_PREDICTION, ent_dev, rel_dev, grad_ent_dev, grad_rel_dev, triples_dev, B,
                                    step, loss_dev);
    if (int rc = check_candidate_step(h, RELATION_PREDICTION, s, loss_reduction, [&]() -> int {
            if (!(weight > 0.f && weight <= FLT_MAX))
                return fail(KGE_ERR_INVALID_ARGUMENT, "kge_one_vs_all_relation_step: weight must be finite and > 0, got %g",
                            (double)weight);
            return KGE_OK;
        }, false, ws_dev, ws_bytes))
        return rc;
    if (B == 0) return KGE_OK;
    cudaStream_t st = (cudaStream_t)stream;
    CandidateQueries q;
    if (int rc = start_candidate_step(h, RELATION_PREDICTION, loss_reduction, ws_dev, step, st, s, &q)) return rc;
    s.side = KGE_SIDE_P;
    s.col = 1;
    s.q = q.qs;
    s.weight = weight;
    KGE_CUDA(launch_relation_prediction_side(s, q.qs, h->L.halves, st, q.drop.cand ? &q.drop : nullptr),
             "kge_one_vs_all_relation_step");
    return KGE_OK;
}

extern "C" int64_t kge_k_vs_all_workspace_bytes(const kge_handle *h, int64_t B)
{
    return candidate_workspace_bytes(h, K_VS_ALL, B);
}

extern "C" int kge_k_vs_all_step(kge_handle *h, int32_t side, int32_t loss_reduction, float label_smoothing,
                                 const float *ent_dev, const float *rel_dev, float *grad_ent_dev, float *grad_rel_dev,
                                 const int32_t *queries_dev, int64_t B, const int64_t *label_offsets_dev,
                                 const int32_t *label_ids_dev, uint64_t step, double *loss_dev, void *ws_dev,
                                 int64_t ws_bytes, void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_k_vs_all_step");
    OneVsAllSide s = candidate_side(h, K_VS_ALL, ent_dev, rel_dev, grad_ent_dev, grad_rel_dev, queries_dev,
                                    B, step, loss_dev);
    if (int rc = check_candidate_step(h, K_VS_ALL, s, loss_reduction, [&]() -> int {
            if (side != KGE_ONE_VS_ALL_S && side != KGE_ONE_VS_ALL_O)
                return fail(KGE_ERR_INVALID_ARGUMENT, "kge_k_vs_all_step: side must be KGE_ONE_VS_ALL_S or "
                                                      "KGE_ONE_VS_ALL_O, got %d", side);
            if (!(label_smoothing >= 0.f && label_smoothing < 1.f))
                return fail(KGE_ERR_INVALID_ARGUMENT, "kge_k_vs_all_step: label_smoothing must be in [0, 1), got %g",
                            (double)label_smoothing);
            return KGE_OK;
        }, !label_offsets_dev || !label_ids_dev, ws_dev, ws_bytes))
        return rc;
    if (B == 0) return KGE_OK;
    cudaStream_t st = (cudaStream_t)stream;
    CandidateQueries q;
    if (int rc = start_candidate_step(h, K_VS_ALL, loss_reduction, ws_dev, step, st, s, &q)) return rc;
    s.side = side == KGE_ONE_VS_ALL_S ? KGE_SIDE_S : KGE_SIDE_O;
    s.col = side == KGE_ONE_VS_ALL_S ? 0 : 2;
    s.q = side == KGE_ONE_VS_ALL_S ? q.qs : q.qo;
    s.label_off = (const long long *)label_offsets_dev;
    s.label_ids = label_ids_dev;
    s.y0 = (float)((double)label_smoothing / (double)h->cfg.n_ent);
    s.y1 = (float)(1.0 - (double)label_smoothing);
    KGE_CUDA(launch_k_vs_all_side(s, h->L.halves, st, q.drop.cand ? &q.drop : nullptr), "kge_k_vs_all_step");
    return KGE_OK;
}

// Embedding dropout of the three all-candidate steps (kge_dropout.cu; DESIGN.md 3.19).  Allowed while a deferred
// step is pending: it only changes what the next all-candidate step computes.
extern "C" int kge_set_embedding_dropout(kge_handle *h, float p_ent, float p_rel, uint64_t seed)
{
    if (!h) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_set_embedding_dropout: null handle");
    if (!(p_ent >= 0.f && p_ent < 1.f) || !(p_rel >= 0.f && p_rel < 1.f))
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_set_embedding_dropout: p_ent and p_rel must be in [0, 1), got %g and %g",
                    (double)p_ent, (double)p_rel);
    h->drop_p_ent = p_ent == 0.f ? 0.f : p_ent;  // -0 clears too
    h->drop_p_rel = p_rel == 0.f ? 0.f : p_rel;
    h->drop_seed = seed;
    return KGE_OK;
}

// ---- the N3 regulariser of a step's positives (kge_reg_n3.cu) -----------------------------------------------------

extern "C" int64_t kge_n3_workspace_bytes(const kge_handle *h)
{
    if (!h) return 0;
    return (int64_t)((4 * (size_t)(h->cfg.n_ent + h->cfg.n_rel) + 15) / 16 * 16);
}

// Allowed while a KGE_STEP_FUSED_DEFER step is pending: it only adds into gradient rows, which the pending step's owner
// kernel (kge_optimizer_step_deferred) reads for every row of the [ent | rel] block afterwards, and it uses its own
// workspace, not the training workspace that holds the pending sum.
extern "C" int kge_n3_step(kge_handle *h, float lambda_ent, float lambda_rel, const float *ent_dev, const float *rel_dev,
                           float *grad_ent_dev, float *grad_rel_dev, const int32_t *triples_dev, int64_t B, uint64_t step,
                           double *loss_dev, void *ws_dev, int64_t ws_bytes, void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_n3_step");
    if (!(lambda_ent >= 0.f && lambda_ent <= FLT_MAX) || !(lambda_rel >= 0.f && lambda_rel <= FLT_MAX) ||
        (lambda_ent == 0.f && lambda_rel == 0.f))
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_n3_step: lambda_ent and lambda_rel must be finite and >= 0, and not both 0; "
                                              "got %g and %g", (double)lambda_ent, (double)lambda_rel);
    if (lambda_rel > 0.f && h->cfg.scoring == KGE_ROTATE)
        return fail(KGE_ERR_UNSUPPORTED, "kge_n3_step: RotatE's relation rows are phases, not embeddings: N3 applies to its "
                                         "entity table only (lambda_rel = 0)");
    if (B < 0) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_n3_step: B < 0");
    if (B == 0) return KGE_OK;
    if (!triples_dev || (lambda_ent > 0.f && (!ent_dev || !grad_ent_dev)) || (lambda_rel > 0.f && (!rel_dev || !grad_rel_dev)))
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_n3_step: null table, gradient or triples");
    if (int rc = check_workspace(ws_dev, ws_bytes, kge_n3_workspace_bytes(h), 16, "kge_n3_step", "kge_n3_workspace_bytes"))
        return rc;
    N3Params p;
    memset(&p, 0, sizeof(p));
    p.ent = ent_dev;
    p.rel = rel_dev;
    p.grad_ent = grad_ent_dev;
    p.grad_rel = grad_rel_dev;
    p.triples = triples_dev;
    p.B = B;
    p.n_ent = h->cfg.n_ent;
    p.n_rel = h->cfg.n_rel;
    p.row_begin = lambda_ent > 0.f ? 0 : h->cfg.n_ent;
    p.row_end = lambda_rel > 0.f ? h->cfg.n_ent + h->cfg.n_rel : h->cfg.n_ent;
    p.kp = h->L.kp;
    p.ld = h->L.ld;
    p.lambda_ent = lambda_ent;
    p.lambda_rel = lambda_rel;
    p.lambda3_ent = (float)(3.0 * (double)lambda_ent);
    p.lambda3_rel = (float)(3.0 * (double)lambda_rel);
    p.cnt = (int *)ws_dev;
    p.loss = loss_dev;
    // the rows the step's positives use are already looked up; stamped anyway (only while the entity buffer is set, as
    // by every other step entry point)
    p.stamp = kge_step_stamp(step);
    p.stamp_ent = h->stamp_ent;
    p.stamp_rel = h->stamp_ent ? h->stamp_rel : nullptr;
    KGE_CUDA(launch_n3(p, h->L.halves, h->sm_count, (cudaStream_t)stream), "kge_n3_step");
    return KGE_OK;
}

// ---- the DURA regulariser of a step's positives (kge_reg_dura.cu) -------------------------------------------------

// Allowed while a KGE_STEP_FUSED_DEFER step is pending, like kge_n3_step: it only adds into gradient rows, which the
// pending step's owner kernel (kge_optimizer_step_deferred) reads for every row of the [ent | rel] block afterwards, and it
// takes no workspace.
extern "C" int kge_dura_step(kge_handle *h, float weight_norm, float weight_prod, const float *ent_dev, const float *rel_dev,
                             float *grad_ent_dev, float *grad_rel_dev, const int32_t *triples_dev, int64_t B, uint64_t step,
                             double *loss_dev, void *stream)
{
    KGE_CHECK_HANDLE(h, "kge_dura_step");
    if (h->cfg.scoring == KGE_TRANSE || h->cfg.scoring == KGE_ROTATE)
        return fail(KGE_ERR_UNSUPPORTED, "kge_dura_step: DURA is defined for the tensor-factorisation scores (DistMult, "
                                         "ComplEx, HolE); not for TransE or RotatE");
    if (!(weight_norm >= 0.f && weight_norm <= FLT_MAX) || !(weight_prod >= 0.f && weight_prod <= FLT_MAX) ||
        (weight_norm == 0.f && weight_prod == 0.f))
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_dura_step: weight_norm and weight_prod must be finite and >= 0, and not "
                                              "both 0; got %g and %g", (double)weight_norm, (double)weight_prod);
    if (B < 0) return fail(KGE_ERR_INVALID_ARGUMENT, "kge_dura_step: B < 0");
    if (B == 0) return KGE_OK;
    if (!triples_dev || !ent_dev || !grad_ent_dev || (weight_prod > 0.f && (!rel_dev || !grad_rel_dev)))
        return fail(KGE_ERR_INVALID_ARGUMENT, "kge_dura_step: null table, gradient or triples");
    DuraParams p;
    memset(&p, 0, sizeof(p));
    p.ent = ent_dev;
    p.rel = rel_dev;
    p.grad_ent = grad_ent_dev;
    p.grad_rel = grad_rel_dev;
    p.triples = triples_dev;
    p.B = B;
    p.kp = h->L.kp;
    p.ld = h->L.ld;
    p.w_norm = weight_norm;
    p.w_prod = weight_prod;
    p.w_prod2 = 2.f * weight_prod;
    p.loss = loss_dev;
    // stamped only while the entity buffer is set, as by every other step entry point
    p.stamp = kge_step_stamp(step);
    p.stamp_ent = h->stamp_ent;
    p.stamp_rel = h->stamp_ent ? h->stamp_rel : nullptr;
    KGE_CUDA(launch_dura(p, h->L.halves, (cudaStream_t)stream), "kge_dura_step");
    return KGE_OK;
}
