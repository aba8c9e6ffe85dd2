/* knn_oracle.c -- TEST INFRASTRUCTURE: the canonical distance chains of kge_knn / kge_radius_neighbors in C.
 *
 * Built with -ffp-contract=off (knn_oracle.py), so the only fused operation is the explicit fmaf; every other
 * operation is one correctly rounded fp32 operation, in ascending column order, exactly as include/kge_b200.h states:
 *   euclidean: acc = +0; for c: t = q_c - x_c; acc = fmaf(t, t, acc); d = sqrtf(acc)
 *   manhattan: acc = +0; for c: acc = acc + |q_c - x_c|;               d = acc
 * A numpy restatement cannot reproduce fmaf (a double product + sum rounds twice).
 */
#include <math.h>
#include <stdint.h>

/* out[i, j] = d(A[i], Bm[j]) for A [na, K], Bm [nb, K] (row-major fp32); metric 0 = euclidean, 1 = manhattan */
void kgeo_distances(int metric, int64_t K, const float *A, int64_t na, const float *Bm, int64_t nb, float *out)
{
    for (int64_t i = 0; i < na; ++i) {
        const float *q = A + i * K;
        for (int64_t j = 0; j < nb; ++j) {
            const float *x = Bm + j * K;
            float acc = 0.f;
            if (metric == 0) {
                for (int64_t c = 0; c < K; ++c) {
                    const float t = q[c] - x[c];
                    acc = fmaf(t, t, acc);
                }
                acc = sqrtf(acc);
            } else {
                for (int64_t c = 0; c < K; ++c) acc = acc + fabsf(q[c] - x[c]);
            }
            out[i * nb + j] = acc;
        }
    }
}
