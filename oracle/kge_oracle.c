/*
 * kge_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Plain-C CPU restatement of the scoring / ranking half of AmpliGraph's hot
 * path.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference leg may load this library; the product (ampligraph_b200/)
 * never does.
 *
 * What it restates (paths under ampligraph/latent_features/ of the reference):
 *   scoring  layers/scoring/TransE.py:37-114, DistMult.py:34-99,
 *            ComplEx.py:39-151, HolE.py:31-89, RotatE.py:62-217
 *   ranks    layers/scoring/AbstractScoringLayer.py:156-422
 *            (+1 and 's+o' handling live in models/ScoringBasedEmbeddingModel.py
 *            :1459-1463,:1684 and are applied by the caller)
 *   lookup   layers/encoding/EmbeddingLookupLayer.py:332-334
 *   corrupt  layers/corruption_generation/CorruptionGenerationLayerTrain.py:35-94
 *            (structure only; TF's stateful RNG stream cannot be restated)
 *
 * Parity status: PINNED for scores, ranks, lookup by the reference's own
 * golden vectors (tests/golden/reference_kats.json, extracted from the
 * reference's tests by tests/golden/extract_reference_kats.py).  The
 * floating-point *summation order* of TensorFlow's reductions is not
 * observable from the reference sources, so this file fixes a canonical
 * order -- ascending row index, one fused multiply-add per term where
 * written as fmaf() -- and the CUDA ranking kernels follow the same order,
 * which is what makes ranks bit-exact between the two.  Compile with
 * -ffp-contract=off so that only the explicit fmaf() calls fuse.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum { KGEO_TRANSE = 0, KGEO_DISTMULT = 1, KGEO_COMPLEX = 2, KGEO_HOLE = 3, KGEO_ROTATE = 4 };
enum { KGEO_SIDE_S = 0, KGEO_SIDE_O = 1 };
enum { KGEO_WORST = 0, KGEO_BEST = 1, KGEO_MIDDLE = 2 };

/* ---- canonical sin/cos ------------------------------------------------
 * RotatE.py:97-98 takes tf.cos / tf.sin of a float32 phase.  libm and CUDA
 * disagree in the last ulp, which would flip int32(score*1000) at
 * quantisation boundaries, so both sides use this deterministic routine:
 * double-precision Cody-Waite reduction by pi/2 and Taylor polynomials,
 * every operation an IEEE fma/mul/add, result rounded once to float.
 * Accuracy ~1e-16 relative before the final rounding (checked against libm
 * in tests/test_oracle.py). */
static const double KGEO_2_OVER_PI = 6.36619772367581382433e-01;
static const double KGEO_PIO2_HI = 1.57079632679489655800e+00;
static const double KGEO_PIO2_LO = 6.12323399573676603587e-17;

static double kgeo_poly_sin(double r)
{
    /* r - r^3/3! + r^5/5! ... up to r^17 */
    double r2 = r * r;
    double p = 2.81145725434552075980e-15;           /*  1/17! */
    p = fma(p, r2, -7.64716373181981647590e-13);     /* -1/15! */
    p = fma(p, r2, 1.60590438368216145994e-10);      /*  1/13! */
    p = fma(p, r2, -2.50521083854417187751e-08);     /* -1/11! */
    p = fma(p, r2, 2.75573192239858906526e-06);      /*  1/9!  */
    p = fma(p, r2, -1.98412698412698412698e-04);     /* -1/7!  */
    p = fma(p, r2, 8.33333333333333333333e-03);      /*  1/5!  */
    p = fma(p, r2, -1.66666666666666666667e-01);     /* -1/3!  */
    return fma(r * r2, p, r);
}

static double kgeo_poly_cos(double r)
{
    /* 1 - r^2/2! + r^4/4! ... up to r^16 */
    double r2 = r * r;
    double p = 4.77947733238738529744e-14;           /*  1/16! */
    p = fma(p, r2, -1.14707455977297247139e-11);     /* -1/14! */
    p = fma(p, r2, 2.08767569878680989792e-09);      /*  1/12! */
    p = fma(p, r2, -2.75573192239858906526e-07);     /* -1/10! */
    p = fma(p, r2, 2.48015873015873015873e-05);      /*  1/8!  */
    p = fma(p, r2, -1.38888888888888888889e-03);     /* -1/6!  */
    p = fma(p, r2, 4.16666666666666666667e-02);      /*  1/4!  */
    p = fma(p, r2, -5.00000000000000000000e-01);     /* -1/2!  */
    return fma(r2, p, 1.0);
}

void kgeo_sincosf(float xf, float *s_out, float *c_out)
{
    double x = (double)xf;
    double n = rint(x * KGEO_2_OVER_PI);
    double r = fma(-n, KGEO_PIO2_HI, x);
    r = fma(-n, KGEO_PIO2_LO, r);
    double s = kgeo_poly_sin(r), c = kgeo_poly_cos(r);
    long long q = (long long)n & 3;
    double ss, cc;
    switch (q) {
    case 0: ss = s; cc = c; break;
    case 1: ss = c; cc = -s; break;
    case 2: ss = -s; cc = -c; break;
    default: ss = -c; cc = s; break;
    }
    *s_out = (float)ss;
    *c_out = (float)cc;
}

/* RotatE.py:96-98: embedding_range = (6/(K*R))**0.5 (python double);
 * phase = theta / (embedding_range/pi) with the divisor converted to fp32. */
float kgeo_rotate_divisor(int K, int max_rel_size)
{
    double range = sqrt(6.0 / ((double)K * (double)max_rel_size));
    return (float)(range / 3.14159265358979323846);
}

/* HolE.py:45: (2 / (internal_k / 2)) as a python double, cast to fp32 by TF. */
float kgeo_hole_scale(int K) { return (float)(2.0 / ((double)K / 2.0)); }

/* ---- triple score: _compute_scores ------------------------------------ */
float kgeo_score_triple(int model, int K, int max_rel_size, const float *s, const float *p,
                        const float *o)
{
    int h = K / 2;
    float acc = 0.0f;
    switch (model) {
    case KGEO_TRANSE: /* TransE.py:51-53  -||s+p-o||_1 */
        for (int d = 0; d < K; ++d) acc = acc + fabsf((s[d] + p[d]) - o[d]);
        return -acc;
    case KGEO_DISTMULT: /* DistMult.py:48  sum(s*p*o) */
        for (int d = 0; d < K; ++d) acc = fmaf(s[d] * p[d], o[d], acc);
        return acc;
    case KGEO_COMPLEX:
    case KGEO_HOLE: /* ComplEx.py:57-62 */
        for (int d = 0; d < h; ++d) {
            float A = fmaf(p[h + d], o[h + d], p[d] * o[d]);
            acc = fmaf(s[d], A, acc);
        }
        for (int d = 0; d < h; ++d) {
            float B = fmaf(-p[h + d], o[d], p[d] * o[h + d]);
            acc = fmaf(s[h + d], B, acc);
        }
        return model == KGEO_HOLE ? kgeo_hole_scale(K) * acc : acc;
    case KGEO_ROTATE: { /* RotatE.py:78-104 */
        float div = kgeo_rotate_divisor(K, max_rel_size);
        for (int d = 0; d < h; ++d) {
            float pr, pi_;
            kgeo_sincosf(p[d] / div, &pi_, &pr);
            float re = fmaf(-s[h + d], pi_, s[d] * pr) - o[d];
            float im = fmaf(s[h + d], pr, s[d] * pi_) - o[h + d];
            acc = acc + sqrtf(fmaf(im, im, re * re));
        }
        return -acc;
    }
    }
    return NAN;
}

/* Per-query vector that the corruption score contracts the candidate row
 * with.  qv has K floats.  For RotatE it holds (cos|sin) on the subject side
 * and the rotated subject on the object side. */
static void kgeo_query_vector(int model, int side, int K, int max_rel_size, const float *s,
                              const float *p, const float *o, float *qv)
{
    int h = K / 2;
    switch (model) {
    case KGEO_TRANSE:
        for (int d = 0; d < K; ++d) qv[d] = side == KGEO_SIDE_S ? p[d] - o[d] : s[d] + p[d];
        break;
    case KGEO_DISTMULT:
        for (int d = 0; d < K; ++d) qv[d] = side == KGEO_SIDE_S ? p[d] * o[d] : s[d] * p[d];
        break;
    case KGEO_COMPLEX:
    case KGEO_HOLE:
        for (int d = 0; d < h; ++d) {
            if (side == KGEO_SIDE_S) { /* ComplEx.py:95-108 */
                qv[d] = fmaf(p[h + d], o[h + d], p[d] * o[d]);
                qv[h + d] = fmaf(-p[h + d], o[d], p[d] * o[h + d]);
            } else { /* ComplEx.py:139-150 */
                qv[d] = fmaf(-s[h + d], p[h + d], s[d] * p[d]);
                qv[h + d] = fmaf(s[d], p[h + d], s[h + d] * p[d]);
            }
        }
        break;
    case KGEO_ROTATE: {
        float div = kgeo_rotate_divisor(K, max_rel_size);
        for (int d = 0; d < h; ++d) {
            float pr, pi_;
            kgeo_sincosf(p[d] / div, &pi_, &pr);
            if (side == KGEO_SIDE_S) {
                qv[d] = pr;
                qv[h + d] = pi_;
            } else { /* RotatE.py:208-211 */
                qv[d] = fmaf(-s[h + d], pi_, s[d] * pr);
                qv[h + d] = fmaf(s[h + d], pr, s[d] * pi_);
            }
        }
        break;
    }
    }
}

/* score of one candidate row e for a prepared query (qv, plus o for RotatE
 * subject side): _get_subject_corruption_scores / _get_object_corruption_scores */
static float kgeo_candidate_score(int model, int side, int K, const float *qv, const float *o,
                                  const float *e)
{
    int h = K / 2;
    float acc = 0.0f;
    switch (model) {
    case KGEO_TRANSE: /* TransE.py:78-84 / :107-113 */
        if (side == KGEO_SIDE_S)
            for (int d = 0; d < K; ++d) acc = acc + fabsf(e[d] + qv[d]);
        else
            for (int d = 0; d < K; ++d) acc = acc + fabsf(qv[d] - e[d]);
        return -acc;
    case KGEO_DISTMULT: /* DistMult.py:71-73 / :96-98 */
    case KGEO_COMPLEX:  /* ComplEx.py:95-108 / :139-150 */
    case KGEO_HOLE:
        for (int d = 0; d < K; ++d) acc = fmaf(e[d], qv[d], acc);
        return model == KGEO_HOLE ? kgeo_hole_scale(K) * acc : acc;
    case KGEO_ROTATE:
        for (int d = 0; d < h; ++d) {
            float re, im;
            if (side == KGEO_SIDE_S) { /* RotatE.py:151-163 */
                re = fmaf(-e[h + d], qv[h + d], e[d] * qv[d]) - o[d];
                im = fmaf(e[h + d], qv[d], e[d] * qv[h + d]) - o[h + d];
            } else { /* RotatE.py:208-216 */
                re = qv[d] - e[d];
                im = qv[h + d] - e[h + d];
            }
            acc = acc + sqrtf(fmaf(im, im, re * re));
        }
        return -acc;
    }
    return NAN;
}

/* EmbeddingLookupLayer.py:332-334 */
void kgeo_lookup(const float *table, int64_t ld, int K, const int32_t *ids, int64_t n, float *out)
{
    for (int64_t i = 0; i < n; ++i) memcpy(out + i * K, table + (int64_t)ids[i] * ld, sizeof(float) * K);
}

/* predict path: gather + _compute_scores (ScoringBasedEmbeddingModel.py:1694-1699) */
void kgeo_score_triples(int model, int K, int max_rel_size, const float *ent, const float *rel,
                        int64_t ld, const int32_t *triples, int64_t n, float *out)
{
    for (int64_t i = 0; i < n; ++i)
        out[i] = kgeo_score_triple(model, K, max_rel_size, ent + (int64_t)triples[3 * i] * ld,
                                   rel + (int64_t)triples[3 * i + 1] * ld,
                                   ent + (int64_t)triples[3 * i + 2] * ld);
}

/* full [b, m] corruption-score matrix for one side (for the KATs) */
void kgeo_corruption_scores(int model, int side, int K, int max_rel_size, const float *es,
                            const float *ep, const float *eo, int64_t b, const float *cand,
                            int64_t ld, int64_t m, float *out)
{
    float *qv = (float *)malloc(sizeof(float) * (size_t)K);
    for (int64_t i = 0; i < b; ++i) {
        kgeo_query_vector(model, side, K, max_rel_size, es + i * K, ep + i * K, eo + i * K, qv);
        for (int64_t c = 0; c < m; ++c)
            out[i * m + c] = kgeo_candidate_score(model, side, K, qv, eo + i * K, cand + c * ld);
    }
    free(qv);
}

static int32_t kgeo_quant(float score) { return (int32_t)(score * 1000.0f); } /* AbstractScoringLayer.py:11,:201 */

/* AbstractScoringLayer.get_ranks, one side, on already gathered embeddings.
 *   es/ep/eo   [b,K] embeddings of the test triples
 *   cand       [m,ld] candidate rows (ent_matrix); row c has original id start_id + c
 *   filt_off   [b+1] CSR offsets or NULL (no filter); filt_ids = known-true entity ids
 *              (already mapped through mapping_dict by the caller when a subset is used)
 *   out        [b] rank counts BEFORE the caller's +1
 */
void kgeo_ranks_side(int model, int side, int strategy, int K, int max_rel_size, const float *es,
                     const float *ep, const float *eo, int64_t b, const float *cand, int64_t ld,
                     int64_t m, int32_t start_id, int32_t end_id, const int64_t *filt_off,
                     const int32_t *filt_ids, int32_t *out)
{
    float *qv = (float *)malloc(sizeof(float) * (size_t)K);
    for (int64_t i = 0; i < b; ++i) {
        const float *s = es + i * K, *p = ep + i * K, *o = eo + i * K;
        int32_t qpos = kgeo_quant(kgeo_score_triple(model, K, max_rel_size, s, p, o));
        kgeo_query_vector(model, side, K, max_rel_size, s, p, o, qv);
        int32_t gt = 0, ge = 0, eq = 0;
        for (int64_t c = 0; c < m; ++c) {
            int32_t qc = kgeo_quant(kgeo_candidate_score(model, side, K, qv, o, cand + c * ld));
            gt += qpos < qc;
            ge += qpos <= qc;
            eq += qpos == qc;
        }
        int32_t rank;
        if (strategy == KGEO_BEST) rank = gt;                     /* :221-227 */
        else if (strategy == KGEO_MIDDLE) rank = gt + (eq + 1) / 2; /* :232-244 ceil(eq/2) */
        else rank = ge;                                           /* :252-258 */
        if (filt_off) { /* :260-307 -- always '<=' */
            for (int64_t f = filt_off[i]; f < filt_off[i + 1]; ++f) {
                int32_t id = filt_ids[f];
                if (id < start_id || id > end_id) continue; /* :280-288 */
                int32_t qf = kgeo_quant(
                    kgeo_candidate_score(model, side, K, qv, o, cand + (int64_t)(id - start_id) * ld));
                rank -= qpos <= qf;
            }
        }
        out[i] = rank;
    }
    free(qv);
}

/* Convenience: ranks straight from tables + int32 triples, candidates = rows
 * [start_id, end_id] of the entity table (get_emb_matrix_test with one part
 * is start 0, end E-1), or an explicit subset list (cand_ids != NULL, in which
 * case filter ids must already be subset positions). */
void kgeo_rank_triples(int model, int side, int strategy, int K, int max_rel_size,
                       const float *ent, const float *rel, int64_t ld, const int32_t *triples,
                       int64_t b, const int32_t *cand_ids, int64_t n_cand, int32_t start_id,
                       const int64_t *filt_off, const int32_t *filt_ids, int32_t *out)
{
    float *es = (float *)malloc(sizeof(float) * (size_t)(b * K));
    float *ep = (float *)malloc(sizeof(float) * (size_t)(b * K));
    float *eo = (float *)malloc(sizeof(float) * (size_t)(b * K));
    for (int64_t i = 0; i < b; ++i) {
        memcpy(es + i * K, ent + (int64_t)triples[3 * i] * ld, sizeof(float) * K);
        memcpy(ep + i * K, rel + (int64_t)triples[3 * i + 1] * ld, sizeof(float) * K);
        memcpy(eo + i * K, ent + (int64_t)triples[3 * i + 2] * ld, sizeof(float) * K);
    }
    if (cand_ids) {
        float *cand = (float *)malloc(sizeof(float) * (size_t)(n_cand * K));
        for (int64_t c = 0; c < n_cand; ++c)
            memcpy(cand + c * K, ent + (int64_t)cand_ids[c] * ld, sizeof(float) * K);
        kgeo_ranks_side(model, side, strategy, K, max_rel_size, es, ep, eo, b, cand, K, n_cand, 0,
                        (int32_t)(n_cand - 1), filt_off, filt_ids, out);
        free(cand);
    } else {
        kgeo_ranks_side(model, side, strategy, K, max_rel_size, es, ep, eo, b,
                        ent + (int64_t)start_id * ld, ld, n_cand, start_id,
                        (int32_t)(start_id + n_cand - 1), filt_off, filt_ids, out);
    }
    free(es);
    free(ep);
    free(eo);
}

/* CorruptionGenerationLayerTrain.call:52-94 given the two random draws.
 * keep_subj[eta*B] in {0,1}, repl[eta*B] in [0, ent_size); row j*B+i is the
 * j-th corruption of positive i (tf.tile order). */
void kgeo_corrupt(const int32_t *pos, int64_t B, int eta, const uint8_t *keep_subj,
                  const int32_t *repl, int32_t *out)
{
    for (int64_t r = 0; r < B * (int64_t)eta; ++r) {
        int64_t i = r % B;
        int32_t ks = keep_subj[r] ? 1 : 0, ko = 1 - ks;
        out[3 * r + 0] = ks * pos[3 * i + 0] + ko * repl[r];
        out[3 * r + 1] = pos[3 * i + 1];
        out[3 * r + 2] = ko * pos[3 * i + 2] + ks * repl[r];
    }
}
