/*
 * kge_b200.h -- C-ABI of libkge_b200.so, the sm_90a replacement for AmpliGraph's
 * per-batch training step and all-entity ranking step.
 *
 * The reference has no FFI: its boundary is two Python registries and three
 * step closures (SURVEY.md 8b).  Each entry point below names the reference
 * code it replaces (paths under ampligraph/latent_features/ of the reference).
 * A Python maintainer binds these with ctypes (see INTEGRATION.md).
 *
 * Conventions
 *   - plain C types only; every `*_dev` / table / output pointer is a DEVICE
 *     pointer owned by the caller (PyTorch tensors in the shipped facade); the
 *     library borrows it for the duration of the call and allocates nothing
 *     persistent except the small per-handle workspace created by kge_create.
 *   - `stream` is a cudaStream_t passed as void* (NULL = default stream); all
 *     work is stream-ordered; no entry point synchronises the device or allocates
 *     device memory (scratch space is a caller-owned workspace, see kge_rank).
 *   - every entry point that launches work first makes kge_config.device the
 *     current device of the calling thread and restores the previous one on
 *     return, so handles of different GPUs can be driven from one thread.
 *   - return value: 0 = ok, otherwise a kge_status; text via kge_last_error().
 *   - one caller thread per handle; different handles (one per GPU) may be
 *     driven from different threads.
 *
 * Embedding-table layout in HBM ("row-padded split-complex")
 *   A table is [rows, ld] fp32, row-major.  TransE/DistMult rows hold k values
 *   padded with zeros to kp = round_up(k,4) floats (ld = kp).  ComplEx/HolE/
 *   RotatE rows hold the real half then the imaginary half, EACH padded to kp
 *   floats (ld = 2*kp).  Rows are therefore 16-byte multiples, which is what
 *   cp.async.bulk / cp.reduce.async.bulk need.  Pad columns are zero and stay
 *   zero.  kge_pack_rows / kge_unpack_rows convert from/to the reference's
 *   dense [rows, internal_k] layout (EmbeddingLookupLayer.py:194-237).
 */
#ifndef KGE_B200_H
#define KGE_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KGE_B200_ABI_VERSION 2

typedef struct kge_handle kge_handle;

enum kge_status {
    KGE_OK = 0,
    KGE_ERR_INVALID_ARGUMENT = 1, /* facade raises ValueError */
    KGE_ERR_CUDA = 2,             /* facade raises RuntimeError */
    KGE_ERR_UNSUPPORTED = 3       /* facade raises NotImplementedError */
};

/* SCORING_LAYER_REGISTRY names, layers/scoring/AbstractScoringLayer.py:15 */
enum kge_scoring { KGE_TRANSE = 0, KGE_DISTMULT = 1, KGE_COMPLEX = 2, KGE_HOLE = 3, KGE_ROTATE = 4 };

/* LOSS_REGISTRY names, loss_functions.py:17; KGE_LOSS_EXTERNAL = LossFunctionWrapper
 * (:657): the caller differentiates its own loss on the scores and hands back
 * d loss / d score (see kge_train_step). */
enum kge_loss {
    KGE_LOSS_PAIRWISE = 0,
    KGE_LOSS_NLL = 1,
    KGE_LOSS_ABSOLUTE_MARGIN = 2,
    KGE_LOSS_SELF_ADVERSARIAL = 3,
    KGE_LOSS_MULTICLASS_NLL = 4
};
enum kge_reduction { KGE_REDUCE_SUM = 0, KGE_REDUCE_MEAN = 1 }; /* loss_functions.py:124-129 */
enum kge_optimizer {
    KGE_OPT_SGD = 0,
    KGE_OPT_ADAM = 1,
    KGE_OPT_ADAGRAD = 2,
    KGE_OPT_RMSPROP = 3,
    KGE_OPT_ADADELTA = 4,
    KGE_OPT_ADAMAX = 5,
    KGE_OPT_NADAM = 6,
    KGE_OPT_FTRL = 7
};
/* the element of (s, p, o) a ranking / top-k call replaces by its candidates: subject or object (entity rows), or the
 * relation (KGE_SIDE_P, relation prediction: candidates are relation rows, see kge_rank) */
enum kge_side { KGE_SIDE_S = 0, KGE_SIDE_O = 1, KGE_SIDE_P = 2 };
enum kge_rank_strategy { KGE_RANK_WORST = 0, KGE_RANK_BEST = 1, KGE_RANK_MIDDLE = 2 };
/* how kge_rank scores the candidates of DistMult / ComplEx / HolE (the bilinear models, a [b,K]x[K,E] contraction):
 * AUTO = tensor cores (wgmma, split-bf16 operands) decide every (query, candidate) pair whose approximate score is
 * provably on one side of the positive's quantisation bin, the few remaining pairs are re-scored with the exact
 * canonical FP32 chain -- ranks are bit-identical to EXACT, which runs that chain for every pair. */
enum kge_rank_mode { KGE_RANK_MODE_AUTO = 0, KGE_RANK_MODE_EXACT = 1 };
/* initialisers for kge_init_table (tf.keras.initializers the reference accepts, EmbeddingLookupLayer.py:105-129) */
enum kge_init {
    KGE_INIT_UNIFORM = 0,           /* U[a, b) */
    KGE_INIT_NORMAL = 1,            /* N(mean a, stddev b) */
    KGE_INIT_TRUNCATED_NORMAL = 2,  /* N(a, b) resampled until within 2 stddev (Keras TruncatedNormal) */
    KGE_INIT_CONSTANT = 3           /* a */
};
enum kge_step_mode {
    KGE_STEP_FUSED = 0,         /* scores -> built-in loss -> gradients, one kernel */
    KGE_STEP_FORWARD_ONLY = 1,  /* scores only (user-callable loss / FocusE, phase 1) */
    KGE_STEP_BACKWARD_EXT = 2,  /* gradients from caller-supplied dL/dscore (phase 2) */
    KGE_STEP_FUSED_DEFER = 3    /* KGE_STEP_FUSED, but the gradient rows of the replaced entities are left pending in the
                                   training workspace: kge_optimizer_step_deferred adds them and applies the optimizer */
};

/* ScoringBasedEmbeddingModel.__init__ (models/ScoringBasedEmbeddingModel.py:100-171)
 * + compile(loss=...) (:1303) + loss hyper-parameters (loss_functions.py:23-29). */
typedef struct kge_config {
    int32_t struct_size;  /* sizeof(kge_config), ABI guard */
    int32_t scoring;      /* enum kge_scoring */
    int32_t k;            /* user-facing embedding size; internal_k = k or 2k */
    int32_t eta;          /* negatives per positive */
    int64_t n_ent;        /* max_ent_size: rows of ent_emb; corruptions are drawn from [0,n_ent) */
    int64_t n_rel;        /* max_rel_size: rows of rel_emb (RotatE phase normalisation uses it) */
    int32_t loss;         /* enum kge_loss */
    int32_t reduction;    /* enum kge_reduction */
    float margin;         /* pairwise / absolute_margin / self_adversarial */
    float alpha;          /* self_adversarial temperature */
    int32_t device;       /* CUDA device ordinal */
    int32_t neg_group;    /* 0 = auto; >0 forces that many negatives resident per pass (testing) */
    int64_t max_rel_size; /* RotatE phase normalisation sqrt(6/(internal_k*max_rel_size)) (RotatE.py:96,
                             ScoringBasedEmbeddingModel.py:338); 0 = n_rel */
    int32_t rank_mode;    /* enum kge_rank_mode */
    int32_t rank_pair_cap; /* 0 = auto (max(2^20, b*n_cand/16)); >0 caps the list of undecided pairs of the tensor-core
                              filter -- a testing knob for its overflow fallback */
} kge_config;

/* optimizers.get (optimizers.py:255-291) -> tf.keras.optimizers.legacy.{SGD,Adam,Adagrad,RMSprop,Adadelta,Adamax,Nadam,
 * Ftrl};
 * regularizers.LP_regularizer (regularizers.py:14-37) folded into the update.
 * What the two slot buffers of the optimizer calls (slot0 / slot1, [rows, ld], zero-initialised unless noted) hold:
 *   SGD       momentum accumulator (only with momentum != 0) / -
 *   Adam      m / v
 *   Adagrad   accumulator (initial_accumulator_value) / -
 *   RMSprop   ms / mg when centered, the momentum accumulator when momentum != 0, else -
 *             (centered with momentum needs a third slot: refused, KGE_ERR_UNSUPPORTED)
 *   Adadelta  accum / accum_update
 *   Adamax    m / v (the exponentially weighted infinity norm)
 *   Nadam     m / v
 *   Ftrl      accumulator n (initial_accumulator_value) / linear term z
 * Two older layouts are accepted for the kinds they knew; their missing fields read as 0: a config whose struct_size
 * stops before `rho` (the layout before RMSprop, Adadelta and Adamax) for the first three kinds, and one that stops
 * before `l1` (the layout before Nadam and Ftrl) for the first six.
 * Nadam's per-step scalars are the caller's: before each step t (1-based) it forms, in fp32 as Keras' legacy Nadam
 * does (_prepare_local), m_t = b1 (1 - 0.5 * 0.96^(decay t)), m_t1 = b1 (1 - 0.5 * 0.96^(decay (t + 1))), advances its
 * momentum cache c (1.0 before the first step) to s_new = c * m_t, and sets s_next = s_new * m_t1 and
 * v_den = 1 - b2^t; the same values serve both tables of the step (DESIGN.md 3.3). */
typedef struct kge_optimizer_config {
    int32_t struct_size;
    int32_t kind;         /* enum kge_optimizer */
    float learning_rate;  /* default 0.001 (optimizers.py:284) */
    float beta_1, beta_2; /* Adam, Adamax: 0.9, 0.999 */
    float epsilon;        /* 1e-7 */
    float momentum;       /* SGD, RMSprop: 0 */
    float initial_accumulator_value; /* Adagrad: 0.1 */
    int32_t reg_p;        /* 0 = no regulariser, else p of LP (1, 2, 3, ...) */
    float reg_lambda;     /* LP lambda (default 1e-5) */
    int32_t reg_p2;       /* optional second LP term (Keras 'l1_l2' = p 1 + p 2); 0 = none */
    float reg_lambda2;
    float rho;            /* RMSprop: 0.9, Adadelta: 0.95 */
    int32_t centered;     /* RMSprop: 0 */
    float l1;             /* Ftrl l1_regularization_strength: 0 */
    float l2;             /* Ftrl l2_regularization_strength: 0 */
    float l2_shrinkage;   /* Ftrl l2_shrinkage_regularization_strength: 0 (> 0: ApplyFtrlV2) */
    float lr_power;       /* Ftrl learning_rate_power: -0.5 */
    float ftrl_beta;      /* Ftrl beta: 0 (the rule uses l2 + beta / (2 learning_rate)) */
    float nadam_m_t;      /* Nadam, this step's m_t, m_t1, s_new, s_next and v_den (see above) */
    float nadam_m_t1;
    float nadam_s_new;
    float nadam_s_next;
    float nadam_v_den;
} kge_optimizer_config;

const char *kge_last_error(void);
int kge_abi_version(void);

int kge_create(const kge_config *cfg, kge_handle **out);
void kge_destroy(kge_handle *h);

/* layout queries: internal_k (ComplEx.py:37, RotatE.py:57), padded half, row stride */
int32_t kge_internal_k(const kge_handle *h);
int32_t kge_half_stride(const kge_handle *h); /* kp */
int32_t kge_row_stride(const kge_handle *h);  /* ld, floats */

/* dense [rows, internal_k] <-> padded device layout [rows, ld]; both device pointers. */
int kge_pack_rows(kge_handle *h, const float *dense_dev, float *table_dev, int64_t rows, void *stream);
int kge_unpack_rows(kge_handle *h, const float *table_dev, float *dense_dev, int64_t rows, void *stream);

/* EmbeddingLookupLayer.build with the default 'glorot_uniform' initialiser
 * (EmbeddingLookupLayer.py:194-201): U(-l, l), l = sqrt(6/(rows+internal_k)),
 * from a Philox4x32-10 counter stream (TF's own stream is not reproducible). */
int kge_init_glorot_uniform(kge_handle *h, float *table_dev, int64_t rows, uint64_t seed, void *stream);
/* The other initialisers tf.keras.initializers.get resolves for entity_relation_initializer (random_normal,
 * random_uniform, truncated_normal, glorot_normal, he_*, lecun_*, zeros, ones, constant; the fan-dependent ones
 * are reduced to these four kinds by the caller): one Philox4x32-10 draw per element, pads stay 0. */
int kge_init_table(kge_handle *h, float *table_dev, int64_t rows, int32_t kind, float a, float b, uint64_t seed,
                   void *stream);

/* predict_step (ScoringBasedEmbeddingModel.py:1694-1699): gather + _compute_scores. */
int kge_score_triples(kge_handle *h, const float *ent_dev, const float *rel_dev,
                      const int32_t *triples_dev /*[n,3]*/, int64_t n, float *scores_dev /*[n]*/,
                      void *stream);

/* CorruptionGenerationLayerTrain.call (CorruptionGenerationLayerTrain.py:35-94):
 * writes the [eta*B,3] corruption tensor (row j*B+i = j-th corruption of positive i)
 * the fused kernel would draw for (seed, step).  Needed only for inspection / parity. */
int kge_generate_corruptions(kge_handle *h, const int32_t *triples_dev, int64_t B, uint64_t seed,
                             uint64_t step, int32_t *corruptions_dev /*[eta*B,3]*/, void *stream);

/* Host-side replay of that stream -- plain CPU code, no GPU and no handle needed.  The corruption RNG is
 * Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11; the Random123
 * known-answer vectors are checked in tests/test_oracle.py) with counter = (row j*B+i, step) and
 * key = seed: keep_subj = x & 1, replacement id = (y * n_ent) >> 32.  kge_host_corruptions writes the same
 * [eta*B,3] tensor kge_generate_corruptions / the fused kernel produce for (seed, step) on the device, so a
 * run can be audited or reproduced without one (TensorFlow's own stream,
 * CorruptionGenerationLayerTrain.py:55-74, is stateful and not reproducible outside TF). */
void kge_philox4x32_10(const uint32_t ctr[4], const uint32_t key[2], uint32_t out[4]);
int kge_host_corruptions(const int32_t *triples_host /*[B,3]*/, int64_t B, int32_t eta, int64_t n_ent,
                         uint64_t seed, uint64_t step, int32_t *corruptions_host /*[eta*B,3]*/);

/* Negative sampler of sampled training (extension; DESIGN.md 3.18): Bernoulli side choice (Wang et al., AAAI 2014),
 * pseudo-typed pools (PyKEEN's PseudoTypedNegativeSampler) and filtered negatives.  kge_sample_negatives writes the
 * [eta*B] neg_ent_dev / neg_keep_subj_dev arrays kge_train_step takes.  Corruption r = j*B+i (tile order) draws its
 * attempt a from Philox4x32-10 with counter (r_lo, r_hi | a << 24, step_lo, step_hi) and key = seed (attempt 0 is the
 * block kge_generate_corruptions uses):
 *   side    attempt 0 only: keep_subj = x & 1 without thresholds; with them the subject is replaced iff x < thresholds[p]
 *   entity  pool[(y * |pool|) >> 32], the pool of (p, replaced side); all entities [0, n_ent) without pools or where
 *           the pool row is empty
 *   filter  a corruption (s, p, c) (object replaced) or (c, p, o) (subject replaced) whose pair (p * n_ent + kept
 *           entity, c) is in that side's filter arrays is drawn again (entity only) with attempt a + 1 while
 *           a + 1 < max_attempts; after the last attempt it is emitted and *misses_dev is incremented.
 * With every optional array NULL the output is the stream of kge_generate_corruptions.  Deterministic, stream-ordered,
 * allocates nothing. */
typedef struct kge_negative_sampler {
    int32_t struct_size;              /* sizeof(kge_negative_sampler), ABI guard */
    int32_t max_attempts;             /* 1..256 draws of a corruption's entity (1: no re-draw) */
    const uint32_t *thresholds_dev;   /* [n_rel] t_p = floor(2^32 |T_p| / (|H_p| + |T_p|)), or NULL: fair coin */
    const int64_t *sub_pool_off_dev;  /* [n_rel + 1] CSR offsets into sub_pool_ids_dev of each relation's subject pool */
    const int32_t *sub_pool_ids_dev;  /*   (both or neither; NULL: every subject is drawn from all entities) */
    const int64_t *obj_pool_off_dev;  /* the same for the object pools */
    const int32_t *obj_pool_ids_dev;
    int64_t sub_filter_n;             /* known pairs of a replaced subject: key p * n_ent + o, value s; lexsorted */
    const int64_t *sub_filter_keys_dev;
    const int32_t *sub_filter_vals_dev;
    int64_t obj_filter_n;             /* known pairs of a replaced object: key p * n_ent + s, value o; lexsorted */
    const int64_t *obj_filter_keys_dev;
    const int32_t *obj_filter_vals_dev;
} kge_negative_sampler;
/* triples_dev [B,3]; eta from the handle; misses_dev: uint64 counter added to, or NULL.  KGE_ERR_INVALID_ARGUMENT
 * without a launch for a bad struct, max_attempts outside 1..256, pool offsets without ids or the reverse, a filter
 * count < 0 or > 0 without its arrays, B < 0, eta*B >= 2^56, or null triples / outputs when B > 0; B = 0 is a no-op. */
int kge_sample_negatives(kge_handle *h, const kge_negative_sampler *sampler, const int32_t *triples_dev, int64_t B,
                         uint64_t seed, uint64_t step, int32_t *neg_ent_dev, uint8_t *neg_keep_subj_dev,
                         uint64_t *misses_dev, void *stream);

/* NSCaching negative sampling (extension; Zhang, Yao, Shao and Chen, ICDE 2019; DESIGN.md 3.20): per-query caches of
 * high-scoring entities, refreshed each step by importance sampling and drawn from uniformly.  Side 0 (subject replaced)
 * has one cache row per distinct (p, o), side 1 (object replaced) one per distinct (s, p); row r of a side holds
 * count[r] <= N1 distinct ids at ids[r * N1 ..].  kge_nscaching_step runs two phases:
 *   refresh  for every positive i and side with update[i][side] = 1, row = key_rows[i][side]: the candidates
 *            c = 0, 1, ... are the row's count cached ids, then N2 draws e_j = (w * n_ent) >> 32, w word j & 3 of
 *            Philox4x32-10 with counter (row, (j >> 2) | side << 31, step_lo, step_hi) and key
 *            (seed_lo, seed_hi ^ 0x4E534341).  A candidate equal to an earlier one, with a NaN score, or (filter) whose
 *            corrupted triple (s, p, c) / (c, p, o) is a known pair is dropped.  score = kge_corruption_scores' value;
 *            key = fl(score + G), G = -logf(-logf(u)), u = ((w' >> 9) + 0.5) 2^-23, w' word c & 3 of the block with
 *            counter (row, (c >> 2) | 1 << 30 | side << 31, step_lo, step_hi).  The min(N1, valid) candidates with the
 *            largest keys (ties: lower c) are kept, in ascending c, and count is set to their number.
 *   draw     corruption r = j*B + i: v = the block of kge_generate_corruptions, side = keep_subj = x & 1,
 *            n = count[key_rows[i][side]]; replacement ids[row][(y * n) >> 32], or (y * n_ent) >> 32 and
 *            *misses_dev += 1 when n = 0.
 * The rotation table is refreshed from rel_dev for RotatE.  Deterministic, stream-ordered, allocates nothing. */
typedef struct kge_nscaching {
    int32_t struct_size;              /* sizeof(kge_nscaching), ABI guard */
    int32_t cache_size;               /* N1 >= 1 */
    int32_t random_size;              /* N2 >= 1, N1 + N2 <= 512 */
    int32_t pad_;
    int64_t sub_n_keys;               /* rows of the subject-replaced caches (distinct (p, o)) */
    int32_t *sub_ids_dev;             /* [sub_n_keys, N1] */
    int32_t *sub_count_dev;           /* [sub_n_keys] */
    int64_t obj_n_keys;               /* rows of the object-replaced caches (distinct (s, p)) */
    int32_t *obj_ids_dev;             /* [obj_n_keys, N1] */
    int32_t *obj_count_dev;           /* [obj_n_keys] */
    int64_t sub_filter_n;             /* optional filter, as kge_negative_sampler: key p * n_ent + o, value s */
    const int64_t *sub_filter_keys_dev;
    const int32_t *sub_filter_vals_dev;
    int64_t obj_filter_n;             /* key p * n_ent + s, value o */
    const int64_t *obj_filter_keys_dev;
    const int32_t *obj_filter_vals_dev;
} kge_nscaching;
/* ent_dev / rel_dev the tables; triples_dev [B,3]; key_rows_dev int32 [B,2] (row of each side, < that side's n_keys);
 * update_dev uint8 [B,2] (at most one positive per row and step may set it); eta from the handle; neg_ent_dev /
 * neg_keep_subj_dev [eta*B] outputs as kge_sample_negatives'; misses_dev uint64 counter added to, or NULL.
 * KGE_ERR_INVALID_ARGUMENT without a launch for a bad struct, N1 / N2 out of bounds, n_keys < 1 or null cache arrays,
 * a filter count < 0 or > 0 without its arrays, B < 0, eta*B >= 2^56, null pointers when B > 0, or a pending
 * KGE_STEP_FUSED_DEFER step; KGE_ERR_UNSUPPORTED while a row stash is set (row-sharded tables).  B = 0 is a no-op. */
int kge_nscaching_step(kge_handle *h, const kge_nscaching *cache, const float *ent_dev, const float *rel_dev,
                       const int32_t *triples_dev, const int32_t *key_rows_dev, const uint8_t *update_dev, int64_t B,
                       uint64_t seed, uint64_t step, int32_t *neg_ent_dev, uint8_t *neg_keep_subj_dev,
                       uint64_t *misses_dev, void *stream);

/* train_step forward+backward (ScoringBasedEmbeddingModel.py:370-429, call :237-269,
 * Loss.__call__ loss_functions.py:185-225, tape.gradient optimizers.py:166).
 *   triples_dev     [B,3] int32 positives
 *   neg_ent_dev     [eta*B] int32 replacement entity ids in tile order, or NULL to draw
 *                   them in-kernel from Philox(seed, step)
 *   neg_keep_subj_dev [eta*B] uint8, 1 = subject kept / object replaced (the reference's
 *                   keep_subj_mask); must be non-NULL iff neg_ent_dev is
 *   grad_*_dev      [rows, ld] fp32 gradient accumulators, ADDED to (zero them or let
 *                   kge_optimizer_step do it)
 *   loss_dev        double accumulator, += sum over the batch of the per-positive loss
 *                   (FUSED mode only; may be NULL)
 *   scores_pos_dev  [B] (may be NULL); scores_neg_dev [eta*B] tile order (may be NULL):
 *                   written in FUSED and FORWARD_ONLY modes
 *   dpos_dev/dneg_dev  dL/dscore inputs for BACKWARD_EXT mode (else NULL) */
int kge_train_step(kge_handle *h, int32_t mode, const float *ent_dev, const float *rel_dev,
                   float *grad_ent_dev, float *grad_rel_dev, const int32_t *triples_dev, int64_t B,
                   const int32_t *neg_ent_dev, const uint8_t *neg_keep_subj_dev, uint64_t seed,
                   uint64_t step, double *loss_dev, float *scores_pos_dev, float *scores_neg_dev,
                   const float *dpos_dev, const float *dneg_dev, void *stream);

/* Shared negatives (extension; DESIGN.md 3.21; PyTorch-BigGraph, DGL-KE): a sampled training step whose B positives
 * are cut into chunks of C consecutive positives, chunk k = positives [k C, min((k + 1) C, B)), each chunk corrupted
 * against one set of eta candidate entities:
 *   candidate  c_{k,j} = (y * n_ent) >> 32, (x, y, ..) the Philox4x32-10 block of kge_generate_corruptions for
 *              corruption r = j*B + k*C (the chunk's first positive), j = 0..eta-1
 *   side       corruption j of positive i replaces the side the per-positive sampler picks for r = j*B + i:
 *              keep_subj = x & 1 without thresholds, with them the subject is replaced iff x < thresholds[p]
 *   corruption (c_{k,j}, p, o) or (s, p, c_{k,j}); candidates equal to a positive's own entity or to each other are
 *              ordinary corruptions (no filtering)
 * With C = 1 the corruptions are kge_generate_corruptions' (kge_sample_negatives' with thresholds only).  The handle's
 * loss and reduction apply per positive to its eta corruption scores, as in kge_train_step; the gradient of every row
 * the step read (s, p, o of each positive, every candidate) is ADDED to grad_*_dev, the loss to *loss_dev (may be
 * NULL), and the lazy optimizer's stamps are written for those rows.  The rotation table is refreshed from rel_dev for
 * RotatE.
 *   chunk       C >= 1 (C >= B: one chunk)
 *   sampler     only its thresholds_dev is used (max_attempts must be valid); NULL: fair coin
 *   workspace   caller-owned, 16-byte aligned, at least kge_shared_negatives_workspace_bytes(h, B, chunk) bytes
 * KGE_ERR_INVALID_ARGUMENT without a launch for chunk < 1, B < 0, eta*B >= 2^56, null pointers when B > 0, a short
 * or not 16-byte aligned workspace, a bad sampler struct or a pending KGE_STEP_FUSED_DEFER step; KGE_ERR_UNSUPPORTED
 * for a sampler with pools or a filter, while a row stash is set (row-sharded tables) or embedding dropout is set, or
 * when the score and gradient passes would need 2^31 or more CTAs (chunks x ceil(min(C, B) / 16) x ceil(eta / 32)).
 * B = 0 is a no-op.
 * Stream-ordered, allocates nothing. */
int64_t kge_shared_negatives_workspace_bytes(const kge_handle *h, int64_t B, int64_t chunk);
int kge_shared_negatives_step(kge_handle *h, int64_t chunk, const float *ent_dev, const float *rel_dev,
                              float *grad_ent_dev, float *grad_rel_dev, const int32_t *triples_dev, int64_t B,
                              const kge_negative_sampler *sampler, uint64_t seed, uint64_t step, double *loss_dev,
                              void *workspace_dev, int64_t ws_bytes, void *stream);

/* Row-sharded entity table (SURVEY.md 8e, BASELINE configs[3],[4]: |E|*k too large for one GPU).
 * Entity id e lives on rank e / rows_per_shard at local row e % rows_per_shard; every rank's shard
 * [rows_per_shard, ld] and its gradient shard are peer-mapped (torch symmetric memory / cudaIpc /
 * VMM), so ent[q] / grad_ent[q] are valid device pointers on THIS rank for every q. */
typedef struct kge_shard_map {
    int32_t struct_size;
    int32_t world;          /* 1..8 */
    int64_t rows_per_shard;
    const float *ent[8];
    float *grad_ent[8];
    int32_t *stamp_ent[8]; /* optional lazy-optimizer row stamps of every shard (all NULL = off); for any world,
                              world 1 included, they replace the entity stamps of kge_set_row_stamps */
} kge_shard_map;

/* kge_train_step on a row-sharded entity table: the SAME fused kernel, its bulk row gathers and
 * red.global.add.v4 gradient scatters simply address whichever rank owns the row -- the row
 * all-to-all (forward) and gradient all-to-all (backward) SURVEY.md 8e describes happen inside the
 * kernel over NVLink peer memory.  kge_config.n_ent is the GLOBAL entity count.  Relations are
 * replicated (rel_dev / grad_rel_dev local; exchange them with kge_optimizer_step_sharded).
 * The caller brackets it with cross-rank barriers: no rank may gather before every rank's
 * optimizer finished, and no optimizer may start before every rank's scatters are complete. */
/* Optional for kge_train_step_sharded: a caller-owned LOCAL buffer of `rows` table rows ([rows, ld]
 * fp32, rows >= B*eta).  When the corruptions of a positive do not all fit in shared memory the
 * gradient pass needs their rows a second time; with a stash the score pass copies every gathered
 * row into it (cp.async.bulk shared->global) and the gradient pass re-reads the LOCAL copy instead
 * of pulling the row through NVLink again, halving the peer traffic. */
int kge_set_row_stash(kge_handle *h, float *stash_dev, int64_t rows);

/* Hot-entity hint for kge_train_step (optional; results are unchanged up to fp32 summation order).  On a skewed graph a
 * handful of entities occupy a large share of all subject / object slots of a batch, and every such positive adds a full
 * gradient row to the SAME row of grad_ent: tens of thousands of atomics per 128-byte line per step, which the L2
 * serialises per address.  ids_host = the most frequent entities of the training set, most frequent first (HOST array;
 * the first KGE_HOT = 1 is used (a second one measured slower), n = 0 clears the hint): the resident trilinear kernel sums their subject / object gradient rows
 * in registers per warp and scatters each once per launch.  The hint takes effect where positives are assigned to warps by
 * a static stride; where kge_train_step assigns them dynamically (the resident kernel on L2-resident tables, see DESIGN.md
 * 3.2) the imbalance the hint cures does not arise and it is ignored (measured: it would cost 7 %).  The reference has no
 * counterpart (TensorFlow's unsorted_segment_sum deduplicates all rows, optimizers.py:166 -> legacy apply_gradients). */
int kge_set_hot_entities(kge_handle *h, const int32_t *ids_host, int32_t n);
/* Optional training workspace for kge_train_step (results are unchanged up to fp32 summation order).  Where the
 * resident trilinear kernel runs (DistMult / ComplEx / HolE, eta <= 32, one table), a step replaces every entity at least
 * once on average (eta*B >= n_ent: the per-entity sum only pays where replaced entities repeat) and a workspace of at least
 * kge_train_workspace_bytes(h, B) bytes is set, a fused step sums the gradient rows of the replaced entities per entity
 * (bucket the eta*B corruptions by replaced entity, then one warp forms each entity's row and adds it once) instead of
 * scattering every corruption's row with atomics; DESIGN.md 3.2.  kge_train_workspace_bytes returns 0 where the path
 * does not apply (the shape, eta*B >= 2^31, a row stash that covers the step, KGE_B200_TRAIN_KERNEL=general): it is the
 * one decision whether a step buckets.  kge_set_train_workspace zeroes the first bytes of the buffer on `stream`;
 * afterwards the library keeps them zero between steps, so the buffer must not be used for anything else (ws_dev = NULL
 * detaches it).  16-byte aligned.  The environment variable KGE_B200_TRAIN_REPL=scatter keeps the atomic scatter for A/B runs (and makes
 * kge_train_workspace_bytes return 0). */
int64_t kge_train_workspace_bytes(const kge_handle *h, int64_t B);
int kge_set_train_workspace(kge_handle *h, void *ws_dev, int64_t bytes, void *stream);
/* 1 when all 3+eta row windows of a positive stay in shared memory (single gather, the stash is never
 * used), 0 when the kernel works in negative groups / column windows, -1 for a NULL handle. */
int kge_rows_resident(const kge_handle *h);

int kge_train_step_sharded(kge_handle *h, int32_t mode, const kge_shard_map *map, const float *rel_dev,
                           float *grad_rel_dev, const int32_t *triples_dev, int64_t B,
                           const int32_t *neg_ent_dev, const uint8_t *neg_keep_subj_dev, uint64_t seed,
                           uint64_t step, double *loss_dev, float *scores_pos_dev, float *scores_neg_dev,
                           const float *dpos_dev, const float *dneg_dev, void *stream);

/* 1vsAll training (Ruffinelli et al., ICLR 2020; the setting of the reference's multiclass_nll docstring,
 * loss_functions.py:580-590): forward + backward of the multiclass NLL of every positive against EVERY entity, no
 * sampled corruptions.  For each positive (s, p, o) and each side in `sides` (a set of the flags below) the logits are
 * l_e = f(s, p, e) (side o) or f(e, p, o) (side s) for all e in [0, n_ent), the positive's own entity t included once;
 * each is clipped to [-75, 75] (zero gradient outside).  loss_reduction KGE_REDUCE_SUM: logsumexp_e(l_e) - l_t;
 * KGE_REDUCE_MEAN: -log(exp(l_t) / (mean_{e != t} exp(l_e) + exp(l_t))).  Other true triples count as negatives (no
 * filtering).  DistMult, ComplEx and HolE only (KGE_ERR_UNSUPPORTED otherwise); the handle's loss, eta and corruption
 * seed are not used; needs n_ent >= 2 and rows whose 32-query tile fits in shared memory (ld <= about 1600 floats).
 *   grad_*_dev  ADDED to, as by kge_train_step; apply kge_optimizer_step (or _lazy) next
 *   step        the lazy-optimizer stamp (kge_set_row_stamps): every entity row and the relation rows of the batch are
 *               stamped with kge_step_stamp(step)
 *   loss_dev    double accumulator += the sum over positives and sides of the loss (may be NULL)
 *   ws_dev      caller-owned, 16-byte aligned, at least kge_one_vs_all_workspace_bytes(h, B) bytes
 * Refused while a KGE_STEP_FUSED_DEFER step is pending.  Works on one (unsharded) entity table.  DESIGN.md 3.12. */
enum kge_one_vs_all_side { KGE_ONE_VS_ALL_S = 1, KGE_ONE_VS_ALL_O = 2 };
int64_t kge_one_vs_all_workspace_bytes(const kge_handle *h, int64_t B);
int kge_one_vs_all_step(kge_handle *h, int32_t sides, int32_t loss_reduction, const float *ent_dev, const float *rel_dev,
                        float *grad_ent_dev, float *grad_rel_dev, const int32_t *triples_dev, int64_t B, uint64_t step,
                        double *loss_dev, void *ws_dev, int64_t ws_bytes, void *stream);

/* Relation prediction as an auxiliary 1vsAll training objective (Chen, Minervini, Riedel and Stenetorp, AKBC 2021):
 * forward + backward of weight * the multiclass NLL of every positive (s, p, o) against EVERY relation, the term
 * weight * L_p of L = L_s + L_o + weight * L_p (kge_one_vs_all_step gives L_s and L_o).  The logits are
 * l_r = f(s, r, o) = scale * <x_r, Qp(s, o)> for all r in [0, n_rel), Qp = d f / dp (DistMult: s * o; ComplEx / HolE:
 * [s_re o_re + s_im o_im | s_re o_im - s_im o_re]), the positive's own relation p the target; clipping, reductions and
 * gradients as kge_one_vs_all_step's with relations in place of entities (KGE_REDUCE_MEAN averages the exp of the
 * n_rel - 1 negatives).  Other relations that hold for (s, o) count as negatives (no filtering).  DistMult, ComplEx
 * and HolE only (KGE_ERR_UNSUPPORTED otherwise, and for rows too wide for the 1vsAll tiles); needs n_rel >= 2 and a
 * finite weight > 0.  B = 0 is a no-op.
 *   grad_*_dev  ADDED to: every relation row, and the batch's s and o entity rows
 *   step        the lazy-optimizer stamp: every relation row and the batch's s and o rows are stamped with
 *               kge_step_stamp(step) (while an entity stamp buffer is set, as for kge_one_vs_all_step)
 *   loss_dev    double accumulator += weight * the sum over positives of the loss (may be NULL)
 *   ws_dev      caller-owned, 16-byte aligned, at least kge_one_vs_all_relation_workspace_bytes(h, B) bytes
 * The relation gradient rows are summed in a fixed order (bit-for-bit repeatable); the entity rows are added with
 * atomics.  Refused while a KGE_STEP_FUSED_DEFER step is pending.  DESIGN.md 3.14. */
int64_t kge_one_vs_all_relation_workspace_bytes(const kge_handle *h, int64_t B);
int kge_one_vs_all_relation_step(kge_handle *h, float weight, int32_t loss_reduction, const float *ent_dev,
                                 const float *rel_dev, float *grad_ent_dev, float *grad_rel_dev, const int32_t *triples_dev,
                                 int64_t B, uint64_t step, double *loss_dev, void *ws_dev, int64_t ws_bytes, void *stream);

/* KvsAll training (Ruffinelli et al., ICLR 2020): forward + backward of the multi-label binary cross-entropy of B
 * queries against EVERY entity on one side.  Query b is row b of queries_dev [B, 3] = (s, p, o): side
 * KGE_ONE_VS_ALL_O scores l_e = f(s, p, e) (the query is (s, p)), side KGE_ONE_VS_ALL_S scores l_e = f(e, p, o) (the
 * query is (p, o)), for all e in [0, n_ent); the answer column (2 or 0) must hold a valid entity id (it is not scored).
 * Its labels are label_ids_dev[label_offsets_dev[b] .. label_offsets_dev[b + 1]): the offsets are absolute into the
 * id array, and each query's labels are ascending, distinct and in [0, n_ent).  Each logit is clipped to [-75, 75]
 * (zero gradient outside).  Target y'_e = (1 - eps) [e is a label] + eps / n_ent (eps = label_smoothing in [0, 1)).
 * loss = w * sum_e softplus(l_e) - y'_e l_e per query, w = 1 (KGE_REDUCE_SUM) or 1 / n_ent (KGE_REDUCE_MEAN): the
 * reference's nll over every (query, entity) pair.  DistMult, ComplEx and HolE only (KGE_ERR_UNSUPPORTED otherwise); the
 * handle's loss, eta and corruption seed are not used; needs n_ent >= 2 and rows whose 32-query tile fits in shared
 * memory (ld <= about 1600 floats).  B = 0 is a no-op.
 *   grad_*_dev  ADDED to, as by kge_train_step; apply kge_optimizer_step (or _lazy) next
 *   step        the lazy-optimizer stamp: every entity row and the relation rows of the batch are stamped with
 *               kge_step_stamp(step)
 *   loss_dev    double accumulator += the sum over queries of the loss (may be NULL)
 *   ws_dev      caller-owned, 16-byte aligned, at least kge_k_vs_all_workspace_bytes(h, B) bytes
 * Refused while a KGE_STEP_FUSED_DEFER step is pending.  Works on one (unsharded) entity table.  DESIGN.md 3.13. */
int64_t kge_k_vs_all_workspace_bytes(const kge_handle *h, int64_t B);
int kge_k_vs_all_step(kge_handle *h, int32_t side, int32_t loss_reduction, float label_smoothing, const float *ent_dev,
                      const float *rel_dev, float *grad_ent_dev, float *grad_rel_dev, const int32_t *queries_dev, int64_t B,
                      const int64_t *label_offsets_dev, const int32_t *label_ids_dev, uint64_t step, double *loss_dev,
                      void *ws_dev, int64_t ws_bytes, void *stream);

/* Embedding dropout of the all-candidate steps (LibKGE's lookup-embedder dropout; DESIGN.md 3.19).  While p_ent or
 * p_rel is non-zero, kge_one_vs_all_step, kge_one_vs_all_relation_step and kge_k_vs_all_step score and differentiate
 * inverted-dropout copies of the embedding elements they read: x~ = fp32(x * scale) where kept, +0 where dropped,
 * scale = fp32(1 / (1 - p)), p_ent for entity rows and p_rel for relation rows (reciprocal relations' inverse rows
 * included).  The raw element's gradient is fp32(scale * m * gradient of x~).  A side's candidate rows share one mask
 * per call (keyed by row id); each query row of the batch takes its own mask per position b; the sides s, o and p draw
 * independent masks.  Element c (column of the padded row) of row `row` takes word c & 3 of
 * philox4x32_10((row, (c >> 2) | (0x80 | tag) << 24, step_lo, step_hi), (seed_lo, seed_hi)) and is kept iff
 * (word >> 8) >= round(p 2^24), with step the step's `step` argument and tag = 4 side + role (side 1 = s, 2 = o,
 * 3 = p; role 0 the candidates, row = table row; role 1 + j the query's triple column j, row = b).  The logged loss is
 * that of the dropped-out scores.  While it is set, the three workspace sizers add two [n_cand, ld] float tables, and
 * kge_train_step and kge_train_step_sharded are refused with KGE_ERR_UNSUPPORTED (their fused kernels do not apply
 * it); kge_n3_step, kge_dura_step, the optimizer and every ranking, scoring and top-k entry point read the raw tables
 * as before.  p_ent = p_rel = 0 clears it, and the steps then run exactly as without it.
 * KGE_ERR_INVALID_ARGUMENT: p_ent or p_rel NaN, < 0 or >= 1. */
int kge_set_embedding_dropout(kge_handle *h, float p_ent, float p_rel, uint64_t seed);

/* The N3 regulariser (Lacroix, Usunier and Obozinski, ICML 2018, eq. 6) of a step's B positives (s_b, p_b, o_b):
 * L_N3 = lambda_ent * sum_b sum_d (|s_bd|^3 + |o_bd|^3) + lambda_rel * sum_b sum_d |p_bd|^3, duplicates counted every
 * time they occur.  |z_d| is |x[d]| for TransE and DistMult, and the modulus sqrt(x[d]^2 + x[kp + d]^2) for ComplEx,
 * HolE and RotatE; the gradient is 3 lambda |z_d| z_d, component-wise.  Only the rows the positives use get a gradient,
 * so a table regularised with N3 keeps the looked-up-rows optimizer rule.  A table whose lambda is 0 is not read or
 * written and may be passed as NULL (table and gradient).  B = 0 is a no-op.
 *   grad_*_dev  ADDED to, one writer per row (bit-for-bit repeatable); call it after the step's data term(s) and before
 *               the optimizer
 *   step        the lazy-optimizer stamp: the rows with an occurrence are stamped with kge_step_stamp(step) (while an
 *               entity stamp buffer is set, as for kge_train_step)
 *   loss_dev    double accumulator += L_N3 (may be NULL)
 *   ws_dev      caller-owned, 16-byte aligned, at least kge_n3_workspace_bytes(h) = (n_ent + n_rel) * 4 bytes rounded
 *               up to 16: the per-row counts, zeroed by the call
 * KGE_ERR_INVALID_ARGUMENT: a lambda not finite or < 0, both lambdas 0, B < 0, null pointers, a short or misaligned
 * workspace.  KGE_ERR_UNSUPPORTED: lambda_rel > 0 for RotatE (its relation rows are phases).  Unlike the other step
 * entry points it is accepted while a KGE_STEP_FUSED_DEFER step is pending: kge_optimizer_step_deferred reads every
 * gradient row of the block, so the N3 rows added here are part of that update.  The tables are the ones the step
 * trained on (the parameters before the update), whole: row-sharded tables are not supported.  DESIGN.md 3.15. */
int64_t kge_n3_workspace_bytes(const kge_handle *h);
int kge_n3_step(kge_handle *h, float lambda_ent, float lambda_rel, const float *ent_dev, const float *rel_dev,
                float *grad_ent_dev, float *grad_rel_dev, const int32_t *triples_dev, int64_t B, uint64_t step,
                double *loss_dev, void *ws_dev, int64_t ws_bytes, void *stream);

/* The DURA regulariser (Zhang, Cai and Wang, NeurIPS 2020) of a step's B positives (h_b, r_b, t_b):
 * L_DURA = sum_b sum_d [ weight_norm (m_h + m_t) + weight_prod m_r (m_h + m_t) ], m_x = |x_d|^2, duplicates counted every
 * time they occur.  |x_d| is |x[d]| for DistMult and the modulus sqrt(x[d]^2 + x[kp + d]^2) for ComplEx and HolE.  With
 * weight_norm = lambda alpha and weight_prod = lambda beta it is the paper's lambda (alpha (|h|^2 + |t|^2) + beta
 * (|h o r|^2 + |t o conj(r)|^2)); with weight_prod = 0 it is the per-occurrence squared L2 of the entity rows.  The
 * gradient, component-wise on each half: 2 (weight_norm + weight_prod m_r) h_d, the same with t_d, and
 * 2 weight_prod (m_h + m_t) r_d.  Only the rows the positives use get a gradient, so a DURA model keeps the looked-up-rows
 * optimizer rule.  With weight_prod = 0 the relation table is not read or written and may be passed as NULL (table and
 * gradient).  B = 0 is a no-op.
 *   grad_*_dev  ADDED to with red.global.add: the same fp32 sum in any order, but the order is the REDs' arrival order,
 *               so it is bit-for-bit repeatable only where every partial sum is exact (as for kge_train_step's kept
 *               rows); call it after the step's data term(s) and before the optimizer
 *   step        the lazy-optimizer stamp: the positives' entity rows, and their relation rows when weight_prod > 0, are
 *               stamped with kge_step_stamp(step) (while an entity stamp buffer is set, as for kge_train_step)
 *   loss_dev    double accumulator += L_DURA (may be NULL)
 * Refusals, in this order: KGE_ERR_UNSUPPORTED for TransE and RotatE; KGE_ERR_INVALID_ARGUMENT for a weight not finite
 * or < 0, both weights 0, B < 0, then null table, gradient or triples pointers.  Like kge_n3_step it is accepted while a
 * KGE_STEP_FUSED_DEFER step is pending: kge_optimizer_step_deferred reads every gradient row of the block, so the DURA
 * rows added here are part of that update.  The tables are the ones the step trained on (the parameters before the
 * update), whole: row-sharded tables are not supported.  DESIGN.md 3.16. */
int kge_dura_step(kge_handle *h, float weight_norm, float weight_prod, const float *ent_dev, const float *rel_dev,
                  float *grad_ent_dev, float *grad_rel_dev, const int32_t *triples_dev, int64_t B, uint64_t step,
                  double *loss_dev, void *stream);

/* OptimizerWrapper.minimize -> legacy apply_gradients (optimizers.py:136-168) for ONE
 * table (or any row-wise concatenation of tables of the same width and regulariser: the engine passes [ent | rel] as one
 * block, one launch per step), dense semantics, plus the LP regulariser's loss/gradient over the whole table
 * (regularizers.py:14-37; added to the loss at loss_functions.py:215-223).
 *   t            1-based iteration count (Adam bias correction)
 *   slot0/slot1  the kind's slots, as listed at kge_optimizer_config ([rows,ld] or NULL where the kind has none)
 *   reg_loss_dev double accumulator += lambda*sum|x|^p of the PRE-update table (may be NULL)
 * The gradient buffer is zeroed on the way out. */
int kge_optimizer_step(kge_handle *h, const kge_optimizer_config *opt, int64_t t, float *table_dev,
                       float *grad_dev, float *slot0_dev, float *slot1_dev, int64_t rows,
                       double *reg_loss_dev, void *stream);

/* kge_optimizer_step over the [ent | rel] block of a KGE_STEP_FUSED_DEFER step, fused with that step's pending sum of
 * the replaced entities' gradient rows: one warp per row adds the row's bucket (DESIGN.md 3.2) to grad_dev's row,
 * applies the optimizer and the regulariser as kge_optimizer_step does, and zeroes the gradient row.
 *   params_in   the block the step trained on: ent_dev, with rel_dev directly after its n_ent rows.  Only READ.
 *   params_out  a second [rows, ld] block: every element of every row is written (pad columns stay 0), so it needs no
 *               initialisation; the caller uses it as the parameter block from then on (double buffering).
 *   grad_dev    the step's grad_ent_dev, with grad_rel_dev directly after it; zeroed on the way out.
 *   rows        n_ent + n_rel.  slot0/slot1 and reg_loss_dev as in kge_optimizer_step (one regulariser for both tables).
 * Fails with KGE_ERR_INVALID_ARGUMENT if no deferred step is pending or the blocks are not the ones it used.  Refused
 * arguments (KGE_ERR_INVALID_ARGUMENT) launch nothing and leave the step pending, so the call can be repeated; any other
 * outcome, a launch failure included, consumes it.  While a step is pending, kge_train_step and kge_set_train_workspace
 * refuse on the handle.  A step can be deferred exactly where kge_train_workspace_bytes(h, B) > 0 and a workspace of that
 * size is set; elsewhere KGE_STEP_FUSED_DEFER returns KGE_ERR_UNSUPPORTED and launches nothing. */
int kge_optimizer_step_deferred(kge_handle *h, const kge_optimizer_config *opt, int64_t t, const float *params_in,
                                float *params_out, float *grad_dev, float *slot0_dev, float *slot1_dev, int64_t rows,
                                double *reg_loss_dev, void *stream);

/* LAZY optimizer (opt-in extension, NOT the reference's dense rule): only rows touched by the
 * step are read and updated; m, v of untouched rows do not decay and the rows do not move (the
 * semantics of TensorFlow-Addons' LazyAdam).  Needed when the dense pass is unaffordable
 * (BASELINE configs[4]: 80 GB table).  kge_set_row_stamps registers caller-owned int32 [rows]
 * buffers; from then on kge_train_step writes kge_step_stamp(step) into the stamp of every row it
 * looks up (whether or not its summed gradient is 0: the rows TensorFlow lists in the IndexedSlices of
 * tf.nn.embedding_lookup), and kge_optimizer_step_lazy(..., row_stamp_dev, kge_step_stamp(step))
 * updates exactly those rows (and zeroes their gradient rows).  Stamping is on only while the entity
 * buffer is set, so a caller that updates only the relation table lazily registers both.  For
 * RMSprop with momentum and Adamax this IS the reference's rule on a table without a regulariser
 * (ResourceSparseApplyRMSProp, and Adamax's gather / scatter of the looked-up rows). */
int kge_set_row_stamps(kge_handle *h, int32_t *ent_stamps_dev, int32_t *rel_stamps_dev);
int32_t kge_step_stamp(uint64_t step);
int kge_optimizer_step_lazy(kge_handle *h, const kge_optimizer_config *opt, int64_t t, float *table_dev,
                            float *grad_dev, float *slot0_dev, float *slot1_dev, int64_t rows,
                            const int32_t *row_stamp_dev, int32_t stamp, double *reg_loss_dev, void *stream);
/* Nadam's rule on an IndexedSlices gradient (Keras' legacy Nadam, _resource_apply_sparse), the reference's rule for a
 * Nadam table without a regulariser: one dense pass in which EVERY row's m and v decay (m *= b1, v *= b2) and only the
 * rows stamped kge_step_stamp(step) add their gradient terms and move, as kge_optimizer_step moves every row (a stamped
 * row whose summed gradient is exactly 0 still moves; an unstamped row with m != 0 does not).  Unstamped rows' table
 * and gradient rows are not read or written (their gradient is 0 by the stamping contract).  KGE_ERR_UNSUPPORTED for
 * any other kind; KGE_ERR_INVALID_ARGUMENT for a config with a regulariser (a regularised table's gradient is dense:
 * kge_optimizer_step) and for the pointers kge_optimizer_step_lazy refuses. */
int kge_optimizer_step_decay(kge_handle *h, const kge_optimizer_config *opt, int64_t t, float *table_dev,
                             float *grad_dev, float *slot0_dev, float *slot1_dev, int64_t rows,
                             const int32_t *row_stamp_dev, int32_t stamp, void *stream);

/* Data-parallel variant of kge_optimizer_step FUSED with the gradient exchange over NVLink peer
 * memory (the reference has no distributed path; SURVEY.md 8e asks for replicated tables + a
 * gradient all-reduce).  Tables are replicated and every rank holds a full gradient table from its
 * own batch.  Rank `rank` owns rows [row_begin, row_end): it reads that shard of EVERY rank's
 * gradient table through peer pointers, sums in rank order, applies the optimizer (slots cover the
 * shard only: [row_end-row_begin, ld]) and stores the updated rows into EVERY rank's table.
 *   peer_tables / peer_grads  HOST arrays of `world` device pointers, indexed by rank; entry [rank]
 *                             is the local buffer, the others are peer-mapped (cudaIpc / VMM /
 *                             torch symmetric memory) addresses
 * The caller must (1) order it after all ranks' kge_train_step (cross-rank barrier), (2) put a
 * second barrier after it before any rank reads a table again, and (3) zero its own gradient
 * table afterwards.  reg_loss_dev receives this rank's shard of the regulariser loss. */
int kge_optimizer_step_sharded(kge_handle *h, const kge_optimizer_config *opt, int64_t t, int32_t world,
                               int32_t rank, float *const *peer_tables, float *const *peer_grads,
                               float *slot0_shard_dev, float *slot1_shard_dev, int64_t row_begin,
                               int64_t row_end, double *reg_loss_dev, void *stream);

/* ONE-LAUNCH data-parallel step tail: cross-rank flag barrier + gradient reduce-scatter + optimizer on this rank's
 * row shard + parameter all-gather + cross-rank flag barrier, all inside one kernel over NVLink peer memory
 * (replaces: barrier kernel, kge_optimizer_step_sharded x2, barrier kernel, two memsets).
 *   peer_tables[q]  base of rank q's REPLICATED parameter block: rows [0,n_ent) entity table immediately followed by
 *                   rows [n_ent, n_ent+n_rel) relation table (one contiguous [n_ent+n_rel, ld] buffer)
 *   peer_grads[q]   base of rank q's gradient block of THIS step, same shape (its kge_train_step scattered into it)
 *   zero_grads_dev  this rank's OTHER gradient block (gradient blocks are double-buffered: step i scatters into block
 *                   i&1); it is zeroed here for the next step -- every peer finished reading it one step ago -- so
 *                   nobody ever memsets a gradient table.  NULL: skip.
 *   slot*_shard_dev optimizer slots of rows [row_begin, row_end) of the concatenated block only
 *   opt_ent/opt_rel the two tables may carry different regularisers (EmbeddingLookupLayer.py:131-155)
 *   table_mc_dev / grads_mc_dev  NULL, or the NVLS MULTICAST mappings of the parameter block and of this step's gradient
 *                   block (torch symmetric memory: multicast_ptr): the gradient shard is then reduced inside the NVSwitch
 *                   (multimem.ld_reduce) and the updated rows are broadcast by it (multimem.st) -- 1/N of a block per
 *                   rank per direction over the links instead of (N-1)/N; peer_tables/peer_grads are still required
 *                   (local reads, fallback)
 *   peer_flags[q]   base of rank q's flag pad: 2*world uint32, zero-initialised once, peer-mapped like the tables
 *   token           strictly increasing per call (e.g. the step count t): flags are never reset
 *   phases          bit 0: wait until every rank entered this call (= finished its kge_train_step) before reading
 *                   gradients; bit 1: before returning control to the stream, wait until every rank delivered its
 *                   rows (so the next kernel on this stream may read the tables).  3 = both (the normal case).
 * Stream order on each rank must be: kge_train_step(step i) -> this call.  No other synchronisation is needed. */
int kge_optimizer_step_exchange(kge_handle *h, const kge_optimizer_config *opt_ent,
                                const kge_optimizer_config *opt_rel, int64_t t, int32_t world, int32_t rank,
                                float *const *peer_tables, float *const *peer_grads, float *table_mc_dev,
                                const float *grads_mc_dev, float *zero_grads_dev,
                                float *slot0_shard_dev, float *slot1_shard_dev, int64_t row_begin,
                                int64_t row_end, uint32_t *const *peer_flags, uint32_t token, int32_t phases,
                                double *reg_loss_dev, void *stream);

/* Diagnostics for the call above: stamps_dev = 8 x uint64 of device memory (caller-owned, kept alive) that every
 * following kge_optimizer_step_exchange launch overwrites with %globaltimer nanoseconds at its phase boundaries --
 * [0] CTA 0 enters, [1] CTA 0 zeroed its part of the next gradient block, [2] CTA 0 passed the entry barrier (all ranks
 * arrived), [3] CTA 0 finished its reduce-scatter/optimizer/all-gather share, [4] CTA 0 fenced and reported done,
 * [5] the last CTA of the grid reported done and signals the peers, [6] every peer signalled: the kernel ends.
 * NULL switches tracing off (the default; the kernel then executes no extra stores).  bench.py prints the phase
 * breakdown of the data-parallel step from these. */
int kge_set_exchange_trace(kge_handle *h, uint64_t *stamps_dev);

/* The flag barrier alone (one tiny kernel): signal `token` into slot `slot` (0 or 1) of every rank's flag pad, then
 * wait until all ranks signalled.  Used by the row-sharded trainer around its local optimizer. */
int kge_peer_barrier(kge_handle *h, int32_t world, int32_t rank, uint32_t *const *peer_flags, int32_t slot,
                     uint32_t token, void *stream);

/* test_function / get_ranks (ScoringBasedEmbeddingModel.py:1387-1465,
 * layers/scoring/AbstractScoringLayer.py:156-422) for one corruption side.
 *   cand_ids_dev  NULL: candidates are entity rows [cand_begin, cand_begin+n_cand) of
 *                 ent_dev (get_emb_matrix_test :1329; a row shard when sharded);
 *                 else [n_cand] int32 entity ids (entities_subset, :1634-1643)
 *   filt_off_dev  [b+1] int64 CSR offsets or NULL (unfiltered); filt_idx_dev = candidate
 *                 POSITIONS (entity id when cand_ids_dev is NULL, subset position
 *                 otherwise) of the known-true entities; positions outside
 *                 [cand_begin, cand_begin+n_cand) are ignored (:280-288);
 *                 n_filt = total number of filter entries (= filt_off[b], known to the host)
 *   ranks_dev     [b] int32, += count (so sides can accumulate); the caller adds 1
 *                 (ScoringBasedEmbeddingModel.py:1684).  May be NULL when counts_dev is given.
 *   counts_dev    NULL, or [b,3] int32 raw counters, += {#(q_pos < q_c), #(q_pos == q_c), #filtered}.
 *                 Candidate partitions (row shards, cand_begin chunks) must accumulate THESE and call
 *                 kge_rank_finalize once: 'middle' is best + ceil(equal/2) (:232-244), which is not
 *                 additive over partitions; 'worst'/'best' are, so ranks_dev may be accumulated directly.
 *   workspace_dev caller-owned scratch of at least kge_rank_workspace_bytes(h, b, n_cand) bytes, 1024-byte
 *                 aligned; contents are undefined afterwards.  The library never allocates or synchronises.
 * side = KGE_SIDE_P (relation prediction, (s, ?, o)): the candidates are RELATION rows -- cand_ids_dev holds relation
 *   ids, or the candidates are rows [cand_begin, cand_begin+n_cand) of the relation table (a range beyond n_rel is
 *   refused); filter entries are candidate positions as above.  Column 1 of triples_dev is the positive relation, scored
 *   whether or not it is among the candidates.  A candidate r's score is the canonical triple score of (s, r, o)
 *   (oracle/kge_oracle.c: kgeo_score_triple, the value quantised as the positive's score, bit for bit): the object-side
 *   chain of TransE / DistMult / RotatE with the query vector built from (s, r), the subject-side chain of ComplEx /
 *   HolE with the query vector built from (r, o).  Counting, strategies, filter and counts_dev are those of the entity
 *   sides.  Every rank_mode runs the exact chain: each pair has its own query vector, so the tensor-core filter has no
 *   per-query operand. */
int kge_rank(kge_handle *h, int32_t side, int32_t strategy, const float *ent_dev,
             const float *rel_dev, const int32_t *triples_dev, int64_t b,
             const int32_t *cand_ids_dev, int64_t cand_begin, int64_t n_cand,
             const int64_t *filt_off_dev, const int32_t *filt_idx_dev, int64_t n_filt,
             int32_t *ranks_dev, int32_t *counts_dev, void *workspace_dev, int64_t workspace_bytes,
             void *stream);

/* kge_rank against THIS rank's row shard of a sharded table: query rows are fetched from whichever
 * rank owns them, candidates are the local shard's rows, filter ids are GLOBAL entity ids (those
 * outside the shard are ignored, AbstractScoringLayer.py:280-288).  Sum counts_dev over ranks
 * (int32 all-reduce) and finalize once (ScoringBasedEmbeddingModel.py:1449-1452).  KGE_SIDE_P is refused
 * (KGE_ERR_INVALID_ARGUMENT): the relation table is replicated, never sharded -- rank relations with kge_rank. */
int kge_rank_sharded(kge_handle *h, const kge_shard_map *map, int32_t rank, int32_t side, int32_t strategy,
                     const float *rel_dev, const int32_t *triples_dev, int64_t b,
                     const int64_t *filt_off_dev, const int32_t *filt_idx_dev, int64_t n_filt,
                     int32_t *ranks_dev, int32_t *counts_dev, void *workspace_dev, int64_t workspace_bytes,
                     void *stream);

/* ranks[i] += f_strategy(counts[i]) - filtered[i]  (AbstractScoringLayer.py:218-258, :304-307) */
int kge_rank_finalize(kge_handle *h, const int32_t *counts_dev /*[b,3]*/, int64_t b, int32_t strategy,
                      int32_t *ranks_dev, void *stream);

/* _get_subject_corruption_scores / _get_object_corruption_scores (TransE.py:56-114, DistMult.py:51-99,
 * ComplEx.py:65-151, HolE.py:47-89, RotatE.py:107-217): the [b, n_cand] fp32 score matrix of every candidate
 * substituted on `side`, canonical summation order (the scores kge_rank quantises).  Same candidate
 * addressing and workspace contract as kge_rank; KGE_SIDE_P gives the canonical triple score of every (s, r, o) with
 * r a candidate relation (the relation column of triples_dev is not read). */
int kge_corruption_scores(kge_handle *h, int32_t side, const float *ent_dev, const float *rel_dev,
                          const int32_t *triples_dev, int64_t b, const int32_t *cand_ids_dev,
                          int64_t cand_begin, int64_t n_cand, float *scores_dev /*[b, n_cand]*/,
                          void *workspace_dev, int64_t workspace_bytes, void *stream);

/* Diagnostic for KGE_RANK_MODE_AUTO (used by the tests that pin its error bound): the APPROXIMATE scores of the
 * tensor-core filter pass and the error bound delta the filter assumes for each pair, both [b, n_cand] fp32, in the
 * units of kge_corruption_scores.  The filter is sound iff |approx - kge_corruption_scores| <= delta everywhere.
 * delta is NaN for every pair of a query or 256-candidate tile that holds a NaN or inf entry: no bound, the filter sends
 * all those pairs to its exact refine.
 * KGE_ERR_UNSUPPORTED when the filter does not apply (model, mode, size, or KGE_SIDE_P). */
int kge_rank_filter_probe(kge_handle *h, int32_t side, const float *ent_dev, const float *rel_dev,
                          const int32_t *triples_dev, int64_t b, const int32_t *cand_ids_dev, int64_t cand_begin,
                          int64_t n_cand, float *approx_dev, float *delta_dev, void *workspace_dev,
                          int64_t workspace_bytes, void *stream);

/* bytes of caller-owned scratch kge_rank / kge_rank_sharded / kge_corruption_scores need for b queries
 * against n_cand candidates (query vectors, counters and -- in KGE_RANK_MODE_AUTO for the bilinear models --
 * the split-bf16 copies of the candidate rows and query vectors the tensor-core pass reads).  The size takes no side:
 * it is an upper bound for KGE_SIDE_P too, which uses the same query-side buffers and never the tensor-core part. */
int64_t kge_rank_workspace_bytes(const kge_handle *h, int64_t b, int64_t n_cand);

/* discovery.query_topn (discovery.py:985-1168), batched: the k best candidates on `side` for each of b queries.
 * Candidates, cand_ids / cand_begin / n_cand and the filter CSR (candidate POSITIONS; those are excluded) follow
 * kge_rank, KGE_SIDE_P (the k best relations of each (s, ?, o), candidates relation rows) included.  Every id in
 * triples_dev must be valid; the column of `side` does not affect the result.
 * ids_dev/scores_dev [b,k]: sorted by (score desc, position asc), NaN first; scores are kge_corruption_scores' bit
 * for bit; rows with fewer than k eligible candidates are padded with id -1, score -inf.
 * The reference scores every completed triple on the host and sorts them all (:1143-1168); here the candidates are
 * scored in L2-sized chunks by the exact FP32 chain (in every rank_mode) and merged into a running top-k per query, so
 * no [b, n_cand] matrix exists.  Any 1 <= k works; k > n_cand pads.  workspace_dev: at least
 * kge_topk_workspace_bytes(h, b, n_cand, k) bytes, 1024-byte aligned, contents undefined afterwards. */
int kge_topk(kge_handle *h, int32_t side, const float *ent_dev, const float *rel_dev, const int32_t *triples_dev,
             int64_t b, const int32_t *cand_ids_dev, int64_t cand_begin, int64_t n_cand,
             const int64_t *filt_off_dev, const int32_t *filt_idx_dev, int64_t n_filt, int32_t k,
             int32_t *ids_dev, float *scores_dev, void *workspace_dev, int64_t workspace_bytes, void *stream);
/* bytes of scratch kge_topk needs: query vectors, one [b, C] score chunk (C sized to half the L2, or
 * KGE_B200_TOPK_CHUNK) and the double-buffered running lists (12 bytes per slot, 2 * b * k slots).  The size takes no
 * side: it is an upper bound for KGE_SIDE_P too. */
int64_t kge_topk_workspace_bytes(const kge_handle *h, int64_t b, int64_t n_cand, int32_t k);

/* the same selection over a caller's [b, n] score matrix (positions out); relation completion uses it
 * (discovery.py:1160-1166: argsort of the predicted scores of the R completed triples).  pos_dev/out_dev [b,k], same
 * order and padding (position -1, -inf) as kge_topk; out_dev holds the input values bit for bit. */
int kge_select_topk(kge_handle *h, const float *scores_dev, int64_t b, int64_t n, int32_t k,
                    int32_t *pos_dev, float *out_dev, void *workspace_dev, int64_t workspace_bytes, void *stream);
int64_t kge_select_topk_workspace_bytes(const kge_handle *h, int64_t b, int64_t n, int32_t k);

/* Distances of kge_knn / kge_radius_neighbors, each a fixed chain over the columns in ascending order with query row q
 * and candidate row x, one correctly rounded fp32 operation at a time:
 *   euclidean: acc = +0; for c: t = q_c - x_c; acc = fma(t, t, acc); d = sqrt(acc)
 *   manhattan: acc = +0; for c: acc = acc + |q_c - x_c|;              d = acc
 * Zero columns present in both rows change nothing, so d over a padded table row equals d over its dense
 * get_embeddings row; d(i, j) == d(j, i) bit for bit. */
enum kge_metric { KGE_METRIC_EUCLIDEAN = 0, KGE_METRIC_MANHATTAN = 1 };

/* sklearn NearestNeighbors.kneighbors (discovery.py:1171-1244): the k nearest (farthest = 1: farthest) of the
 * candidate rows of points_dev [n_points, ld] (ld % 4 == 0, 16-byte aligned) for each query row query_ids_dev[i].
 * Candidates (cand_ids_dev or [cand_begin, cand_begin + n_cand)) and the filter CSR of excluded candidate POSITIONS
 * follow kge_topk.  ids_dev/dist_dev [b, k]: distance ascending (farthest: descending), ties by position ascending;
 * distances bit-identical to the canonical chain; short rows padded with id -1, distance +inf (farthest: -inf).
 * Every id on the device must be valid.  The handle supplies the device and the chunk rule of kge_topk (its model
 * plays no part).  workspace_dev: kge_knn_workspace_bytes bytes, 1024-byte aligned, contents undefined afterwards. */
int kge_knn(kge_handle *h, int32_t metric, const float *points_dev, int64_t n_points, int32_t ld,
            const int32_t *query_ids_dev, int64_t b, const int32_t *cand_ids_dev, int64_t cand_begin, int64_t n_cand,
            const int64_t *filt_off_dev, const int32_t *filt_idx_dev, int64_t n_filt, int32_t k, int32_t farthest,
            int32_t *ids_dev, float *dist_dev, void *workspace_dev, int64_t workspace_bytes, void *stream);
int64_t kge_knn_workspace_bytes(const kge_handle *h, int64_t b, int64_t n_cand, int32_t k, int32_t ld);

/* sklearn radius_neighbors: every candidate with d <= radius (inclusive; the same d as kge_knn, bit for bit).
 * nbr_dev == NULL: count pass, writes offsets_dev[1..b] = per-row counts (offsets_dev[0] = 0); the caller turns them
 * into CSR offsets.  nbr_dev != NULL: offsets_dev holds the CSR offsets, nbr_dev[off[i]..off[i+1]) receives row i's
 * candidate ids in ascending position order (deterministic; ids beyond off[i+1] are dropped). */
int kge_radius_neighbors(kge_handle *h, int32_t metric, const float *points_dev, int64_t n_points, int32_t ld,
                         const int32_t *query_ids_dev, int64_t b, const int32_t *cand_ids_dev, int64_t cand_begin,
                         int64_t n_cand, float radius, int64_t *offsets_dev, int32_t *nbr_dev,
                         void *workspace_dev, int64_t workspace_bytes, void *stream);
int64_t kge_radius_workspace_bytes(const kge_handle *h, int64_t b, int64_t n_cand, int32_t ld);

/* DBSCAN without neighbourhood lists: the device half of discovery.find_clusters (discovery.py:546-711) with sklearn's
 * DBSCAN, whose fit runs a radius_neighbors self-join, keeps every neighbourhood and labels the rows in
 * sklearn.cluster._dbscan_inner.dbscan_inner.  With A(i, j) = d(i, j) <= radius (kge_radius_neighbors' test, i = j
 * included) and core(i) = #{j : A(i, j)} >= min_samples, sklearn's labels are: the connected components of the core
 * rows under A, numbered by their smallest core index; a non-core row with a core neighbour takes the component with
 * the smallest such index among its neighbours'; every other row is noise.  The count pass of kge_radius_neighbors
 * gives the cores; the three calls below give the components and the border rows.  Arguments, candidates, the chunk
 * rule and the workspace (kge_radius_workspace_bytes) are those of kge_radius_neighbors; none allocates or
 * synchronises.
 *
 * kge_radius_union: for every in-radius pair (query_ids_dev[i], candidate id c) with different ids, unions the two in
 * the caller's union-find forest parent_dev[n_points] (int32), which starts as parent[x] = x (or is the result of
 * earlier kge_radius_union calls).  A root hooks under the smaller root, so whatever the order of the unions every
 * tree's root is its smallest id: DBSCAN's component seed.  Concurrent calls may share the forest; parent[x] <= x
 * always, and every x's path leads to its root. */
int kge_radius_union(kge_handle *h, int32_t metric, const float *points_dev, int64_t n_points, int32_t ld,
                     const int32_t *query_ids_dev, int64_t b, const int32_t *cand_ids_dev, int64_t cand_begin,
                     int64_t n_cand, float radius, int32_t *parent_dev, void *workspace_dev, int64_t workspace_bytes,
                     void *stream);
/* out_dev[i] = the smallest key_dev[c] over the candidate ids c within the radius of query row query_ids_dev[i], or
 * INT32_MAX if there is none.  key_dev is indexed by id (n_points entries).  DBSCAN's border rows
 * (dbscan_inner's depth-first search reaches a border row first from the cluster with the smallest seed): queries the
 * non-core rows, candidates the core rows, key the flattened forest. */
int kge_radius_min_key(kge_handle *h, int32_t metric, const float *points_dev, int64_t n_points, int32_t ld,
                       const int32_t *query_ids_dev, int64_t b, const int32_t *cand_ids_dev, int64_t cand_begin,
                       int64_t n_cand, float radius, const int32_t *key_dev, int32_t *out_dev, void *workspace_dev,
                       int64_t workspace_bytes, void *stream);
/* parent_dev[x] = root(x) for every x < n (n < 2^31), after the unions (DBSCAN: the component seed of each core row). */
int kge_forest_flatten(kge_handle *h, int32_t *parent_dev, int64_t n, void *stream);

/* Per-node wedge counts of an undirected simple graph: the device half of discovery.generate_candidates' graph
 * strategies (nx.triangles, nx.clustering and nx.square_clustering, discovery.py:457-471).  No handle: the call runs on
 * the calling thread's current device, on `stream`; it neither allocates nor synchronises.
 *
 * The graph is a CSR over n_nodes < 2^31 nodes: offsets_dev int64 [n_nodes + 1], nbr_dev int32 [offsets[n_nodes]],
 * N(v) = nbr[offsets[v], offsets[v + 1]) without repeats and without v itself (each undirected edge in both lists).
 * order_dev int32 [n_nodes] is a permutation of the nodes, the order in which they are taken (heaviest first,
 * e.g. by sum_{u in N(v)} d(u), balances the load; the results do not depend on it).  With d(v) = |N(v)| and
 * P(v, y) = |N(v) & N(y)|, the call writes int64 [n_nodes]:
 *   tri2_dev[v] = sum_{u in N(v)} P(v, u)                         (twice nx.triangles)
 *   sq_dev[v]   = sum_{y != v} P(v, y) (P(v, y) - 1) / 2
 *   pot_dev[v]  = (sum_{u in N(v)} d(u)) (d(v) - 1) - d(v) (d(v) - 1) - tri2[v] - sq[v]
 * so that nx.clustering = tri2 / (d (d - 1)) (0 if tri2 = 0) and nx.square_clustering = sq / pot (0 if d < 2 or
 * pot <= 0), exactly, in float64.  The results are integers and do not depend on scheduling.
 *
 * Workspace: kge_graph_workspace_bytes(n_nodes) bytes, 8-byte aligned, for the current device (a work counter, plus
 * n_nodes int32 counters per CTA when they do not fit in shared memory: 2 CTAs per SM); 0 = invalid n_nodes or a
 * failed device query.  The contents need no initialisation. */
int kge_graph_counts(const int64_t *offsets_dev, const int32_t *nbr_dev, const int32_t *order_dev, int64_t n_nodes,
                     int64_t *tri2_dev, int64_t *sq_dev, int64_t *pot_dev, void *workspace_dev, int64_t workspace_bytes,
                     void *stream);
int64_t kge_graph_workspace_bytes(int64_t n_nodes);

#ifdef __cplusplus
}
#endif
#endif /* KGE_B200_H */
