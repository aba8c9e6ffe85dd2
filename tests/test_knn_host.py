"""Host-side checks of nearest-neighbour / duplicate search: the C restatement of the distance chains
(tests/knn_oracle.c) against scipy, the duplicate fraction find_duplicates bisects over against the reference's
radius_neighbors + frozenset union, and the fp32 rounding of the radius.  No GPU needed."""
import numpy as np
import pytest

from knn_oracle import distances


@pytest.mark.parametrize("K", [4, 28, 64])
@pytest.mark.parametrize("metric,scipy_metric", [("euclidean", "euclidean"), ("manhattan", "cityblock")])
def test_oracle_distances_match_cdist(metric, scipy_metric, K):
    from scipy.spatial.distance import cdist
    rng = np.random.default_rng(K)
    A = rng.uniform(-1, 1, (17, K)).astype(np.float32)
    B = rng.uniform(-1, 1, (29, K)).astype(np.float32)
    got = distances(metric, A, B)
    want = cdist(A.astype(np.float64), B.astype(np.float64), scipy_metric)
    np.testing.assert_allclose(got, want, rtol=1e-6, atol=0)
    # symmetric bit for bit, zero on the diagonal, zero columns are no-ops
    assert (distances(metric, B, A).T.view(np.uint32) == got.view(np.uint32)).all()
    assert (np.diag(distances(metric, A, A)) == 0).all()
    pad = lambda M: np.concatenate([M[:, :K // 2], np.zeros((len(M), 4), np.float32), M[:, K // 2:]], 1)
    assert (distances(metric, pad(A), pad(B)).view(np.uint32) == got.view(np.uint32)).all()


def _reference_fraction(emb, X, metric, tol):
    """discovery.py:939-961 verbatim: radius_neighbors self-join, frozensets of labels, their union over len(emb)."""
    from sklearn.neighbors import NearestNeighbors
    nn = NearestNeighbors(metric=metric, radius=tol)
    nn.fit(emb)
    neighbors = nn.radius_neighbors(emb)[1]
    dups = {frozenset(X[idx] for idx in row) for i, row in enumerate(neighbors) if len(row) > 1}
    return len(set().union(*dups)) / len(emb)


def _d1(emb, metric):
    """nearest-other-row distance (own position excluded), exact on these integer inputs."""
    diff = emb[:, None, :].astype(np.float64) - emb[None, :, :]
    D = np.sqrt((diff ** 2).sum(-1)) if metric == "euclidean" else np.abs(diff).sum(-1)
    np.fill_diagonal(D, np.inf)
    return D.min(1).astype(np.float32), D


@pytest.mark.parametrize("metric", ["euclidean", "manhattan"])
def test_duplicate_fraction_matches_reference(metric):
    """Integer points (euclidean: on one axis, so every distance is an exact integer in any arithmetic), repeated
    labels with identical rows, and distinct labels sharing a row; tolerances below, between and exactly at every
    attained distance."""
    pytest.importorskip("sklearn")
    from ampligraph_b200.discovery import duplicate_fraction
    rng = np.random.default_rng(5)
    n = 60
    if metric == "euclidean":
        emb = np.zeros((n, 3), np.float32)
        emb[:, 1] = rng.integers(0, 40, n)
    else:
        emb = rng.integers(-3, 4, (n, 3)).astype(np.float32)
    X = np.array(["e%d" % i for i in range(n)], dtype=object)
    X[10:14] = "e3"          # repeated label: rows 3, 10..13 are one entity ...
    emb[10:14] = emb[3]      # ... with one embedding
    emb[20] = emb[21]        # two labels on the same point
    d1, D = _d1(emb, metric)
    frac = duplicate_fraction(d1, X.tolist())
    attained = np.unique(D[np.isfinite(D)])
    grid = sorted(set([0.0, 0.5, 1e9] + attained.tolist() + (attained + 0.5).tolist()))
    for tol in grid:
        assert frac(tol) == _reference_fraction(emb, X, metric, tol), tol


def test_duplicate_fraction_triples():
    """mode 't' keys are tuples of the row; repeated triples count once."""
    pytest.importorskip("sklearn")
    from ampligraph_b200.discovery import duplicate_fraction
    X = np.array([["a", "r", "b"], ["a", "r", "b"], ["c", "r", "d"], ["e", "s", "f"]], dtype=object)
    emb = np.array([[0, 0], [0, 0], [3, 0], [9, 0]], np.float32)
    d1, _ = _d1(emb, "euclidean")
    frac = duplicate_fraction(d1, [tuple(r) for r in X])
    assert frac(0.0) == 1 / 4 and frac(3.0) == 2 / 4 and frac(6.0) == 3 / 4
    Xs = np.array(["|".join(r) for r in X], dtype=object)  # the reference's union over equal hashable keys
    for tol in (0.0, 2.9, 3.0, 6.0, 7.0):
        assert frac(tol) == _reference_fraction(emb, Xs, "euclidean", tol)


def test_fp32_floor():
    from ampligraph_b200.engine import fp32_floor
    for x in (0.0, 1.0, 0.1, 1 / 3, 2.5e-8, 123456.789, -0.7, 1e39):
        r = fp32_floor(x)
        assert float(np.float32(r)) == r and r <= x
        with np.errstate(over="ignore"):
            nxt = float(np.nextafter(np.float32(r), np.float32(np.inf)))
        assert nxt > x
    rng = np.random.default_rng(1)
    d = rng.uniform(0, 2, 10000).astype(np.float32)
    for tol in (0.3, 1.0000001, float(d[7])):
        assert ((d <= np.float32(fp32_floor(tol))) == (d.astype(np.float64) <= tol)).all()
