// kge_internal.h -- internal launcher interfaces of libkge_b200 (not part of the C-ABI).
#pragma once
#include "kge_common.cuh"

// per-lane register state grows with NIT (float4 chunks per lane): trade threads for registers
// (RotatE carries 11 float4 vectors of per-positive state per chunk -- cos, sin, o, y = R s, four Z sums, d/dphi: give it more registers)
// (RotatE with 12 warps at 168 registers was measured no faster than 8 warps at 229 on cfg4 before the H100 port)
#define KGE_TRAIN_THREADS(model, nit) ((nit) <= 1 ? 512 : (nit) == 2 ? ((model) == KGE_ROTATE ? 256 : 384) : 256)
#define KGE_MAX_PEERS 8
#define KGE_MIN_RESIDENT_WARPS 8  // fewer warps/SM than this costs more than re-gathering
#define KGE_TARGET_WARPS 10
#define KGE_MIN_RESIDENT_WARPS_WIDE 6  // the fast path on DistMult rows of 257..512 floats (NIT = 4): 6 resident warps beat the grouped general kernel with 8 on cfg3 (measured before the H100 port)

namespace kge {

struct TrainParams {
    const float *ent;   // [n_ent, ld]
    const float *rel;   // [n_rel, ld]; for RotatE the per-step rotation table [cos|sin]
    float *grad_ent;
    float *grad_rel;
    const int32_t *triples;  // [B,3]
    long long B;
    const int32_t *neg_ent;  // [eta*B] or nullptr (Philox)
    const uint8_t *neg_keep; // [eta*B] or nullptr
    unsigned long long seed, step;
    unsigned n_ent;
    int model, eta, kp, ld, nch;  // nch = kp/4 float4 chunks per half
    int G;                        // replaced rows resident per pass
    int nbuf;                     // group buffers per slot (non-resident): 2 = next group prefetched, 1 = fetched on demand
    int wk, n_cb;                 // column window (floats per half) and number of windows per row
    int slot_floats;              // stride between row windows in the shared-memory slot
    int resident;                 // 1: one window, one group, rows stay in place between the passes
    int eta_pad;                  // round_up(eta,4)
    int rows_bytes, region_bytes; // per-warp shared-memory carve-up
    int loss, reduction, mode;
    float margin, alpha, score_scale, inv_div;
    double *loss_out;
    float *scores_pos, *scores_neg;
    const float *dpos, *dneg;
    // row-sharded entity table (shard_world <= 1: single table at ent / grad_ent)
    int shard_world, rows_per_shard;
    const float *ent_shard[KGE_MAX_PEERS];
    float *grad_ent_shard[KGE_MAX_PEERS];
    // lazy optimizer support: rows touched by this step get stamp written (nullptr: off)
    int stamp;
    int *stamp_ent, *stamp_rel;
    int *stamp_ent_shard[KGE_MAX_PEERS];
    int hot_ent[2];  // entities whose subject/object gradient rows are summed per warp before they are scattered (-1: none); fast path only
    float *stash;  // [B, eta, ld] local copy of the replaced rows gathered by the score pass (sharded runs) or nullptr
    unsigned *sched;  // {next positive, retired warps}: dynamic assignment of positives to warps (see next_positive), or nullptr = static stride
    // owner-computes gradient of the replaced rows (kge_train_bucket.cu; fast path only), carved from the caller's training
    // workspace; bk.g == nullptr: the replaced rows' gradients are scattered with REDs instead
    struct Buckets {
        int *cnt;     // [n_ent] corruptions per replaced entity (zero between steps: the scan resets it)
        int *off;     // [n_ent + 1] CSR offsets of each entity's entries
        int *tiles;   // [ceil(n_ent / 8192)] entries per tile of the two-level scan
        int *pos;     // [eta*B] rank of corruption r = j*B+i inside its entity's bucket
        int *eid;     // [eta*B] entry -> replaced entity
        int *other;   // [eta*B] entry -> the positive's entity on the side that was kept
        int *rel;     // [eta*B] entry -> relation id | side << 31 (1: object replaced)
        float *g;     // [eta*B] entry -> scale * dL/dscore of the corruption
    } bk;
};

// Per-warp shared-memory slot of one training kernel (kge_create): warps per CTA, replaced rows per group, and the
// slot's row windows and total bytes.  warps == 0: the kernel does not apply to the handle's shape.
struct TrainSlot {
    int warps, G, rows_bytes, region_bytes;
};

// Every training launcher runs slot.warps warps per CTA on grid = min(occupancy * sm_count, ceil(B / warps));
// p.G / p.rows_bytes / p.region_bytes are the same slot's.
cudaError_t launch_train(const TrainParams &p, int nit, const TrainSlot &slot, int sm_count, cudaStream_t st);
// kge_train_res.cu: the resident trilinear fast path (DistMult / ComplEx / HolE, all rows of a positive resident, eta <= 32, one
// table)
cudaError_t launch_train_res(const TrainParams &p, int nit, const TrainSlot &slot, int sm_count, cudaStream_t st);
// kge_train_bucket.cu: the owner-computes sum of the replaced rows' gradients around launch_train_res (p.bk set):
// before it, bucket the eta*B corruptions by replaced entity (count + scan); after it, one warp per run of entries
// forms each entity's gradient row and adds it to p.grad_ent once
cudaError_t launch_bucket_prepass(const TrainParams &p, cudaStream_t st);
cudaError_t launch_bucket_sum(const TrainParams &p, int nit, cudaStream_t st);
// kge_train_rot.cu: the RotatE fast path (one column window, single table, any eta in groups of p.G with two buffers -- or one
// group when everything fits)
cudaError_t launch_train_rot(const TrainParams &p, int nit, const TrainSlot &slot, int sm_count, cudaStream_t st);
cudaError_t launch_rotation_table(const float *rel, float *rot, long long n_rel, int kp, int ld, float div,
                                  cudaStream_t st);
cudaError_t launch_corruptions(const int32_t *triples, long long B, int eta, unsigned long long seed,
                               unsigned long long step, unsigned n_ent, int32_t *out, cudaStream_t st);

// kge_negatives.cu: the negative sampler (kge_sample_negatives).  Arrays indexed [side] are [0] for a replaced subject
// and [1] for a replaced object (= keep_subj).
struct NegativeParams {
    const int32_t *triples;  // [B, 3]
    long long B;
    int eta, max_attempts;   // 1 <= max_attempts <= 256
    unsigned n_ent;
    unsigned long long seed, step;
    const uint32_t *thr;            // [n_rel] Bernoulli thresholds, or nullptr: fair coin
    const long long *pool_off[2];   // [n_rel + 1] pool CSR offsets of each side, or nullptr: all entities
    const int32_t *pool_ids[2];
    long long filt_n[2];            // known (key, value) pairs of each side (0: that side is not filtered)
    const long long *filt_keys[2];  // p * n_ent + kept entity, lexsorted with the values
    const int32_t *filt_vals[2];    // the replaced entity
    int32_t *neg_ent;               // [eta * B]
    uint8_t *neg_keep;              // [eta * B]
    unsigned long long *misses;     // += corruptions still known after the last attempt, or nullptr
};
cudaError_t launch_negatives(const NegativeParams &p, int sm_count, cudaStream_t st);

// kge_nscaching.cu: NSCaching (kge_nscaching_step), the refresh of the batch's cache rows, then the draw.  [side] as in
// NegativeParams: [0] the subject-replaced caches (one row per (p, o)), [1] the object-replaced ones (one per (s, p)).
struct NSCacheParams {
    const float *ent, *rel;    // rel: the rotation table for RotatE
    const int32_t *triples;    // [B, 3]
    const int32_t *key_rows;   // [B, 2] cache row of positive i on each side
    const uint8_t *update;     // [B, 2] 1: positive i refreshes that row this step
    long long B;
    int model, kp, ld, eta;
    int n1, n2;                // cache size and random candidates per refresh (n1, n2 >= 1, n1 + n2 <= 512)
    unsigned n_ent;
    float scale;               // HolE's score scale
    unsigned long long seed, step;
    int32_t *ids[2];           // [n_keys, n1]
    int32_t *count[2];         // [n_keys]
    long long filt_n[2];       // known (key, value) pairs of each side, as NegativeParams (0: not filtered)
    const long long *filt_keys[2];
    const int32_t *filt_vals[2];
    int32_t *neg_ent;          // [eta * B]
    uint8_t *neg_keep;         // [eta * B]
    unsigned long long *misses;  // += corruptions drawn from an empty row, or nullptr
};
size_t nscaching_smem_bytes(int ld, int n1, int n2);
cudaError_t launch_nscaching(const NSCacheParams &p, int sm_count, cudaStream_t st);

// kge_train_shared.cu: sampled training with shared negatives (kge_shared_negatives_step).  t carries the tables,
// triples, Philox key, loss and stamps as for the fused step (t.neg_ent and the slot fields are not read).
struct SharedNegParams {
    TrainParams t;
    long long chunk;           // C >= 1 positives per chunk
    const uint32_t *thr;       // [n_rel] Bernoulli side thresholds, or nullptr: fair coin
    float *sc;                 // [B, eta] workspace: scores, then dL/dscore
    uint8_t *keep;             // [B, eta] workspace: side of each corruption (1: object replaced)
    float *pos;                // [B] workspace: the positive's score, then dL/dP
    long long n_chunks, n_ps;  // chunks, and positive slices per chunk, of the score and gradient grids
    int n_jt;                  // candidate tiles
};
// CTAs of the score and gradient passes for (B, chunk, eta); fills q's grid fields when q != nullptr
long long shared_negatives_grid(long long B, long long chunk, int eta, SharedNegParams *q);
// the score, loss and gradient passes, on st
cudaError_t launch_shared_negatives(const SharedNegParams &q, int sm_count, cudaStream_t st);

// kge_train_1vsall.cu: one side of a 1vsAll multiclass-NLL step of the trilinear models (kge_one_vs_all_step)
struct OneVsAllSide {
    const float *q;          // [B, ld] query vectors of the side (launch_rank_prepare: qvec_s for side s, qvec_o for o;
                             // side p: Qp(s, o) of launch_relation_prediction_side)
    const float *ent, *rel;  // [n_ent, ld], [n_rel, ld]
    float *grad_ent, *grad_rel;
    const float *cand;       // [n_cand, ld] candidate rows: ent (sides s, o) or rel (side p)
    float *grad_cand;        // their gradient rows: grad_ent or grad_rel
    const int32_t *triples;  // [B, 3]
    long long B, n_cand;
    int side, col;           // KGE_SIDE_S / KGE_SIDE_O / KGE_SIDE_P; the triple column of the positive's own candidate
    int kp, ld, nsplit;      // nsplit = one_vs_all_splits(B, n_cand) candidate ranges per query tile
    float scale, w;          // HolE's score scale (1 otherwise); weight of a negative's exp (1 or 1 / (n_cand - 1));
                             // KvsAll: weight of every element (1 or 1 / n_ent)
    float weight;            // 1vsAll: the side's weight on its loss and dL/dl (1 for sides s and o; lambda for side p)
    int xsplit;              // dX query-tile ranges per candidate tile: 1 adds to grad_cand directly, > 1 writes
                             // [xsplit, n_cand, ld] partial rows to pgx, summed in split order by launch_grad_passes
    double *loss;            // += sum of the row losses, or nullptr
    int stamp;
    int *stamp_rel;          // lazy-optimizer stamps of the relation rows, or nullptr (sides s, o: the batch's rows)
    int *stamp_ent;          // side p: lazy-optimizer stamps of the entity rows (the batch's s and o rows), or nullptr
    // workspace: [nsplit, B] partial maxima and sums; [B] l_t, max and 1 / D per row (1vsAll only); [nsplit, B, ld]
    // partial Gq rows
    float *pm, *pz, *lt, *row_m, *row_inv, *pgq;
    float *pgx;              // [xsplit, n_cand, ld] partial candidate gradient rows (xsplit > 1 only)
    // KvsAll: the labels of query b are label_ids[label_off[b] .. label_off[b + 1]) (ascending, distinct, < n_ent);
    // target of an entity: y0 = eps / n_ent, plus y1 = 1 - eps for a label
    const long long *label_off;
    const int32_t *label_ids;
    float y0, y1;
};
// kge_dropout.cu: embedding dropout of one side of an all-candidate step (kge_set_embedding_dropout; DESIGN.md 3.19).
// Element c of row `row` under stream tag `tag` takes word c & 3 of philox4x32_10((row, (c >> 2) | (0x80 | tag) << 24,
// step_lo, step_hi), (seed_lo, seed_hi)) and is kept iff (word >> 8) >= t; a kept element is fp32(x * scale), a
// dropped one +0.  tag = 4 side + role: role 0 the candidate rows (row = table row), 1 + j the query's triple column j
// (row = batch position).
struct SideDropout {
    uint64_t seed, step;
    uint32_t t_ent, t_rel;    // keep thresholds of the entity and relation rows (0: keep every element)
    float scale_ent, scale_rel;
    float *cand;              // [n_cand, ld] workspace: the side's dropped candidate table
    float *grad_cand;         // [n_cand, ld] workspace: the candidates' gradient wrt their dropped copies
};
// Writes the dropped candidate table, zeroes grad_cand, writes q[b] from the dropped query rows, and points s.cand,
// s.grad_cand and s.q at them (s.side, s.triples, s.ent, s.rel set; s.cand / s.grad_cand still the raw rows)
cudaError_t launch_dropout_prepare(OneVsAllSide &s, const SideDropout &d, float *q, int halves, cudaStream_t st);
// After the dX pass: adds scale * m times grad_cand to the raw candidate gradient rows, then runs the chain pass on the
// dropped query rows, with each row's own mask on the gradient it adds
cudaError_t launch_dropout_finish(const OneVsAllSide &s, const SideDropout &d, int halves, cudaStream_t st);

int one_vs_all_splits(long long B, long long n_ent);
size_t one_vs_all_smem_bytes(int ld);  // dynamic shared memory of the dQ and dX passes
size_t k_vs_all_smem_bytes(int ld);    // the same with KvsAll's label masks
// drop: the side's embedding dropout, or nullptr (the passes read the raw tables)
cudaError_t launch_one_vs_all_side(const OneVsAllSide &s, int halves, cudaStream_t st, const SideDropout *drop = nullptr);
// one side of a KvsAll multi-label step (kge_k_vs_all_step): s.triples are the [B, 3] queries, s.label_* set
cudaError_t launch_k_vs_all_side(const OneVsAllSide &s, int halves, cudaStream_t st, const SideDropout *drop = nullptr);
cudaError_t launch_one_vs_all_stamps(int *stamp_ent, long long n_ent, int stamp, cudaStream_t st);
// relation prediction as a 1vsAll side (kge_one_vs_all_relation_step): s.side = KGE_SIDE_P, s.cand = rel, s.n_cand =
// n_rel, s.q = qp; writes qp[b] = Qp(s_b, o_b) = d f(s_b, p, o_b) / dp, then runs the 1vsAll passes with dX split
// s.xsplit ways over the query tiles (partials in s.pgx), and a chain pass that adds d/ds and d/do to grad_ent
cudaError_t launch_relation_prediction_side(const OneVsAllSide &s, float *qp, int halves, cudaStream_t st,
                                            const SideDropout *drop = nullptr);

// kge_reg_n3.cu: the N3 regulariser of a step's positives (kge_n3_step)
struct N3Params {
    const float *ent, *rel;         // [n_ent, ld], [n_rel, ld] (nullptr for a table whose lambda is 0)
    float *grad_ent, *grad_rel;
    const int32_t *triples;         // [B, 3]
    long long B, n_ent, n_rel;
    long long row_begin, row_end;   // the rows of the [ent | rel] block with lambda > 0
    int kp, ld;
    float lambda_ent, lambda_rel;   // lambda of each table (0: not regularised)
    float lambda3_ent, lambda3_rel; // 3 * lambda, rounded once
    int *cnt;                       // [n_ent + n_rel] occurrences per row (workspace; zeroed by launch_n3)
    double *loss;                   // += L_N3, or nullptr
    int stamp;
    int *stamp_ent, *stamp_rel;     // lazy-optimizer stamps of the rows with c > 0, or nullptr
};
// memset of p.cnt, the count pass and the apply pass, on st
cudaError_t launch_n3(const N3Params &p, int halves, int sm_count, cudaStream_t st);

// kge_reg_dura.cu: the DURA regulariser of a step's positives (kge_dura_step)
struct DuraParams {
    const float *ent, *rel;         // [n_ent, ld], [n_rel, ld] (rel: nullptr allowed when w_prod is 0)
    float *grad_ent, *grad_rel;
    const int32_t *triples;         // [B, 3]
    long long B;
    int kp, ld;
    float w_norm, w_prod;           // lambda * alpha, lambda * beta
    float w_prod2;                  // 2 * w_prod (exact)
    double *loss;                   // += L_DURA, or nullptr
    int stamp;
    int *stamp_ent, *stamp_rel;     // lazy-optimizer stamps of the positives' rows, or nullptr
};
// one thread per (positive, float4 chunk of a half), gradients by RED, on st
cudaError_t launch_dura(const DuraParams &p, int halves, cudaStream_t st);

// kge_misc.cu
cudaError_t launch_score_triples(const Layout &L, int nit, const float *ent, const float *rel_or_rot,
                                 const int32_t *triples, long long n, float scale, float *out, int sm_count,
                                 cudaStream_t st);
cudaError_t launch_pack(const Layout &L, const float *src, float *dst, long long rows, bool unpack, cudaStream_t st);
cudaError_t launch_glorot(const Layout &L, float *table, long long rows, unsigned long long seed, cudaStream_t st);
cudaError_t launch_init_table(const Layout &L, float *table, long long rows, int kind, float a, float b,
                              unsigned long long seed, cudaStream_t st);

// kge_optim.cu
struct RegParams {  // lambda*sum|x|^p (+ optional second term: Keras 'l1_l2')
    int p, p2;
    float lambda, lambda2;
};
struct OptimParams {
    int kind;
    float lr, lr_t, beta1, beta2, eps, momentum;
    RegParams reg;
    float rho;     // RMSprop / Adadelta decay
    int centered;  // RMSprop
};
// What Nadam and Ftrl read beyond OptimParams, and Nadam's row-decay mode.  Every optimizer kernel takes it as its LAST
// parameter, so the parameters of the kinds before them kept their offsets (and those instantiations their code).
struct OptimStep {
    float l1, l2x2, shrinkx2, lr_power;  // Ftrl: l1, 2 * (l2 + beta / (2 lr)), 2 * l2_shrinkage, learning_rate_power
    float one_m_mt, m_t1, one_m_snew, one_m_snext, v_den;  // Nadam: 1 - m_t, m_t1, 1 - s_new, 1 - s_next, 1 - b2^t
    const int *row_stamp;  // Nadam's IndexedSlices rule (dense kernel only): a row whose stamp != stamp only decays m and
    int stamp, ld4;        // v; nullptr: every row moves.  ld4 = float4s per row
};
struct ExchangeParams {  // kge_optimizer_step_exchange
    int world, rank, phases;
    float *table[KGE_MAX_PEERS];        // [ent|rel] parameter block of every rank
    const float *grad[KGE_MAX_PEERS];   // this step's gradient block of every rank
    unsigned *flags[KGE_MAX_PEERS];     // flag pad of every rank: 2*world uint32
    float *table_mc;                    // NVLS: multicast mapping of the parameter block / this step's gradient block
    const float *grad_mc;               // (both non-null: reduce and broadcast inside the switch), else nullptr
    unsigned token;
    float *zero_grad;                   // local: next step's gradient block, zeroed here (or nullptr)
    long long total4;                   // float4s in one block
    long long off4, n4;                 // this rank's shard
    long long ent4;                     // float4s of the entity part (regulariser switch point)
    RegParams reg_ent, reg_rel;
    float *slot0, *slot1;
    double *reg_loss;
    unsigned *done_counter;             // handle-owned device counter (last-CTA detection), self-resetting
    unsigned long long *trace;          // nullptr or 8 x uint64 phase stamps (kge_set_exchange_trace)
};
cudaError_t launch_optimizer(const OptimParams &o, const OptimStep &os, float *table, float *grad, float *slot0, float *slot1,
                             long long n_floats, double *reg_loss, int sm_count, cudaStream_t st);
cudaError_t launch_optimizer_lazy(const OptimParams &o, const OptimStep &os, float *table, float *grad, float *slot0, float *slot1,
                                  long long rows, int ld, const int *row_stamp, int stamp, double *reg_loss,
                                  int sm_count, cudaStream_t st);
// tables/grads: HOST arrays of `world` device pointers (own rank first is NOT required; index = rank)
cudaError_t launch_optimizer_sharded(const OptimParams &o, const OptimStep &os, int world, int rank, float *const *tables, float *const *grads,
                                     float *slot0, float *slot1, long long off_floats, long long n_floats,
                                     double *reg_loss, int sm_count, cudaStream_t st);
cudaError_t launch_optimizer_exchange(const OptimParams &o, const OptimStep &os, const ExchangeParams &x, int sm_count, cudaStream_t st);
cudaError_t launch_peer_barrier(int world, int rank, unsigned *const *flags, int slot, unsigned token, cudaStream_t st);
// kge_train_bucket.cu: the same per-entity sum with the dense optimizer as its epilogue, one warp per row of the
// [ent | rel] block (rows = n_ent + n_rel; p.ent / p.rel and p.grad_ent / p.grad_rel are the two parts of `in` and `grad`):
// reads `in`, writes every element of `out`, updates the slots in place and zeroes `grad`
cudaError_t launch_bucket_sum_optimizer(const TrainParams &p, int nit, const OptimParams &o, const OptimStep &os, const float *in, float *out,
                                        float *grad, float *slot0, float *slot1, long long rows, double *reg_loss,
                                        cudaStream_t st);

// kge_rank.cu
struct ShardView {  // row-sharded entity table seen through peer pointers (world <= 1: not sharded)
    int world, rows_per_shard;
    const float *ent[KGE_MAX_PEERS];
};
struct RankParams {
    Layout L;
    int side, strategy;
    const float *ent;      // [n_ent, ld]
    const float *qvec;     // [b, ld] prepared query vectors for this side
    const float *qaux;     // [b, ld] object rows (RotatE subject side) or nullptr
    const int32_t *qpos;   // [b] quantised positive scores
    const int32_t *cand_ids;  // nullptr or [n_cand]
    long long cand_begin, n_cand, b;
    long long filt_base;   // subtracted from filter ids (global id of the local shard's first row)
    float scale;           // HolE
    float *scores;         // nullptr, or [b, n_cand] output of every candidate's score (kge_corruption_scores)
    const unsigned *gate;  // nullptr, or device counter: kge_rank_dot_kernel only runs when *gate > gate_cap (overflow fallback
    unsigned gate_cap;     // of the tensor-core filter, kge_rank_tc.cu)
};
cudaError_t launch_rank_prepare(const Layout &L, const ShardView &sv, const float *ent, const float *rel, const float *rot,
                                const int32_t *triples, long long b, float scale, float *qvec_s, float *qvec_o,
                                float *qaux, int32_t *qpos, cudaStream_t st);
// cnt = [b,3] int32 workspace: #(qpos < qc), #(qpos == qc), #filtered
cudaError_t launch_rank_count(const RankParams &p, int32_t *cnt, cudaStream_t st);
// the same with the chain chosen by the caller (an OP_* of kge_rank_common.cuh) instead of by (model, side):
// kge_knn / kge_radius_neighbors score points with OP_L2_SUB / OP_L1_SUB; only p.L.ld is read for the non-RotatE ops
cudaError_t launch_rank_count_op(const RankParams &p, int op, int32_t *cnt, cudaStream_t st);
cudaError_t launch_rank_filter_n(const RankParams &p, const long long *filt_off, const int32_t *filt_idx,
                                 long long n_pairs, int32_t *cnt, int sm_count, cudaStream_t st);
cudaError_t launch_rank_finalize(const int32_t *cnt, long long b, int strategy, int32_t *ranks, cudaStream_t st);
cudaError_t launch_rank_accumulate(const int32_t *cnt, long long b, int32_t *counts, cudaStream_t st);  // counts += cnt

// kge_rank_rel.cu: the relation side (KGE_SIDE_P).  Candidates are rows of rel (the relation table, or RotatE's rotation
// table) through p.cand_ids / p.cand_begin; each query's s and o rows are those of triples[i] in p.ent; p.qpos as
// prepared by launch_rank_prepare; p.qvec / p.qaux are not read.  Same counter and p.scores contract as
// launch_rank_count / launch_rank_filter_n.
cudaError_t launch_rank_rel_count(const RankParams &p, const float *rel, const int32_t *triples, int32_t *cnt, cudaStream_t st);
cudaError_t launch_rank_rel_filter(const RankParams &p, const float *rel, const int32_t *triples, const long long *filt_off,
                                   const int32_t *filt_idx, long long n_pairs, int32_t *cnt, int sm_count, cudaStream_t st);

// kge_topk.cu: running top-k per query over chunks of candidate scores (ordering contract: see the file)
struct TopkSelectParams {
    const float *scores;                 // [b, ld]: this chunk's scores in columns [0, n)
    long long ld, n, base;               // row stride, columns, candidate position of column 0
    long long b;
    int k;
    const long long *filt_off;           // [b+1] CSR offsets or nullptr; filt_idx - filt_shift = candidate positions
    const int32_t *filt_idx;             // to exclude (outside [0, n_cand): ignored)
    long long filt_shift;
    unsigned long long *keys;            // [2, b, k] sorted keys of the running lists (double-buffered)
    float *vals;                         // [2, b, k] their raw scores
    int2 *state;                         // [b] {entries, current buffer}; zero before the first chunk
};
cudaError_t launch_topk_select(const TopkSelectParams &p, cudaStream_t st);
// negate: write -value (padding +inf) instead of the stored value (padding -inf)
cudaError_t launch_topk_write(const int2 *state, const unsigned long long *keys, const float *vals, long long b, int k,
                              const int32_t *cand_ids, long long cand_begin, int32_t *ids, float *out, cudaStream_t st,
                              bool negate = false);

// kge_knn.cu: nearest-neighbour and radius search over the rows of a point matrix (scored by launch_rank_count_op)
// qvec[i, :] = points[query_ids[i], :] for i < b (ld floats, ld % 4 == 0)
cudaError_t launch_knn_gather(const float *points, int ld, const int32_t *query_ids, long long b, float *qvec, cudaStream_t st);
// x = -x over n floats (farthest: turns the chunk's -d into +d, so the select keeps the largest distances)
cudaError_t launch_knn_negate(float *x, long long n, cudaStream_t st);
// one CTA per query row of a [b, ld] chunk of -d scores, columns [0, n) = candidate positions base + c:
// off == nullptr (count): cursor[q] += #{c : d <= radius};
// off != nullptr (emit): the positions' ids (cand_ids[pos] or cand_begin + pos) go to nbr[off[q] + cursor[q] ...] in
// ascending position order and cursor[q] advances (writes beyond off[q + 1] are dropped)
cudaError_t launch_radius_chunk(const float *chunk, long long ld, long long n, long long base, long long b, float radius,
                                const int32_t *cand_ids, long long cand_begin, long long *cursor, const long long *off,
                                int32_t *nbr, cudaStream_t st);
// offsets[0] = 0, offsets[1 + q] = cursor[q]
cudaError_t launch_radius_counts(const long long *cursor, long long b, long long *offsets, cudaStream_t st);

// kge_cluster.cu: the DBSCAN epilogues over the same [b, ld] chunks of -d (columns [0, n) = positions base + c) and
// the union-find forest parent[] they build (invariants in the file's header)
// union(query_ids[q], id(pos)) for every in-radius pair with different ids
cudaError_t launch_radius_union_chunk(const float *chunk, long long ld, long long n, long long base, long long b,
                                      float radius, const int32_t *query_ids, const int32_t *cand_ids,
                                      long long cand_begin, int32_t *parent, cudaStream_t st);
// out[0..b) = INT32_MAX, before the first chunk of launch_radius_min_key_chunk
cudaError_t launch_min_key_init(int32_t *out, long long b, cudaStream_t st);
// out[q] = min(out[q], key[id(pos)] over the in-radius positions)
cudaError_t launch_radius_min_key_chunk(const float *chunk, long long ld, long long n, long long base, long long b,
                                        float radius, const int32_t *cand_ids, long long cand_begin,
                                        const int32_t *key, int32_t *out, cudaStream_t st);
// parent[x] = root(x) for x < n
cudaError_t launch_forest_flatten(int32_t *parent, long long n, cudaStream_t st);

// kge_graph.cu: per-node wedge counts of an undirected simple graph in CSR (definitions in the file's header), on the
// current device.  The workspace (8-byte aligned) holds the work counter and, when n int32 counters do not fit in
// shared memory, one such slice per CTA; graph_workspace_bytes returns 0 for n < 0 or on a device query failure.
long long graph_workspace_bytes(long long n);
cudaError_t launch_graph_counts(const long long *off, const int32_t *nbr, const int32_t *order, long long n,
                                void *workspace, long long *tri2, long long *sq, long long *pot, cudaStream_t st);

// kge_rank_tc.cu: tensor-core filter + exact refine for the bilinear models
struct RankTcLayout {  // carve-up of the tensor-core part of the caller's workspace
    int nkb, n_qb, n_ct;
    unsigned pair_cap;
    size_t off_a, off_b, off_thr, off_tnorm, off_count, off_pairs, bytes;
};
bool rank_tc_applicable(const Layout &L, int side, long long b, long long n_cand);
RankTcLayout rank_tc_layout(const Layout &L, long long b, long long n_cand, int pair_cap_override);
// same contract as launch_rank_count (cnt[3q+0] += #greater, cnt[3q+1] += #equal), bit-identical results.
// probe_a/probe_d != nullptr: diagnostic run -- write approximate scores and assumed error bounds [b, n_cand], count nothing
cudaError_t launch_rank_count_tc(const RankParams &p, const RankTcLayout &w, void *ws, int32_t *cnt, int sm_count, cudaStream_t st,
                                 float *probe_a = nullptr, float *probe_d = nullptr);

}  // namespace kge
