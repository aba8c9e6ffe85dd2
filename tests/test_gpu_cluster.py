"""GPU tests of DBSCAN: KGEEngine.dbscan (kge_radius_neighbors' count pass, kge_radius_union, kge_forest_flatten and
kge_radius_min_key of csrc/kge_cluster.cu) and the discovery facade find_clusters.

The oracle is sklearn's DBSCAN(metric="precomputed") on the C restatement of the distance chains
(tests/knn_oracle.c), passed as fp64: a float32 matrix compared with a Python float would round eps to fp32 and could
move the boundary.  Labels must be equal, and core must equal counts >= min_samples."""
import numpy as np
import pytest
import torch

from knn_oracle import distances as ref_dist

pytestmark = pytest.mark.gpu

METRICS = ["euclidean", "manhattan"]


def _dev(a):
    return torch.as_tensor(a).cuda().contiguous()


def _engine(monkeypatch, chunk=None, kernel=None):
    from ampligraph_b200.engine import KGEEngine
    if chunk is None:
        monkeypatch.delenv("KGE_B200_TOPK_CHUNK", raising=False)
    else:
        monkeypatch.setenv("KGE_B200_TOPK_CHUNK", str(chunk))  # read when the handle is created
    if kernel == "tile":
        monkeypatch.setenv("KGE_B200_RANK_KERNEL", "tile")
    else:
        monkeypatch.delenv("KGE_B200_RANK_KERNEL", raising=False)
    return KGEEngine("TransE", 4, 1, 8, 1)  # the handle only lends its device and chunk rule


def _oracle(D, eps, min_samples):
    from sklearn.cluster import DBSCAN
    labels = DBSCAN(eps=eps, min_samples=min_samples, metric="precomputed").fit_predict(D.astype(np.float64))
    return labels, (D.astype(np.float64) <= eps).sum(1) >= min_samples


def _same(eng, P, metric, eps, min_samples, D=None):
    D = ref_dist(metric, P, P) if D is None else D
    labels, core = (x.cpu().numpy() for x in eng.dbscan(_dev(P), eps, min_samples, metric))
    want, want_core = _oracle(D, eps, min_samples)
    assert labels.dtype == np.int64 and core.dtype == np.bool_
    assert (core == want_core).all(), (eps, min_samples, np.flatnonzero(core != want_core)[:5])
    assert (labels == want).all(), (eps, min_samples, np.flatnonzero(labels != want)[:5])
    return labels


def _blobs(rng, n, ld, centers=8, sigma=0.05, noise=0.1):
    C = rng.uniform(-0.5, 0.5, (centers, ld))
    P = C[rng.integers(0, centers, n)] + rng.normal(0, sigma, (n, ld))
    far = rng.random(n) < noise
    P[far] = rng.uniform(-0.5, 0.5, (int(far.sum()), ld))
    return P.astype(np.float32)


# ---------------------------------------------------------------------------
@pytest.mark.parametrize("kernel", ["pair", "tile"])
@pytest.mark.parametrize("chunk", [None, 256])
@pytest.mark.parametrize("metric", METRICS)
def test_dbscan_vs_oracle(metric, chunk, kernel, monkeypatch):
    """Widths 4, 28 (a column-chunk tail), 400 and 1,200; eps at quantiles of D and equal to an attained distance;
    min_samples 1, 2, 5 and n + 1."""
    rng = np.random.default_rng(11)
    n = 600
    eng = _engine(monkeypatch, chunk, kernel)
    kinds = set()
    for ld in (4, 28, 400, 1200):
        P = _blobs(rng, n, ld)
        D = ref_dist(metric, P, P)
        off = D[~np.eye(n, dtype=bool)]
        for eps in (float(np.quantile(off, 0.02)), float(np.quantile(off, 0.1)), float(np.quantile(off, 0.3)),
                    float(D[3, 77])):
            for ms in (1, 2, 5, n + 1):
                labels = _same(eng, P, metric, eps, ms, D)
                kinds.add("noise" if (labels == -1).all() else "mixed" if (labels == -1).any() else "clustered")
    assert kinds == {"noise", "mixed", "clustered"}
    eng.close()


@pytest.mark.parametrize("metric", METRICS)
def test_dbscan_chain(metric, monkeypatch):
    """5,000 points on a line, neighbours just under eps apart: one component, built through long union paths, with
    the ids in order and shuffled; both ends are border rows at min_samples 3."""
    n, ld = 5000, 4
    P = np.zeros((n, ld), np.float32)
    P[:, 0] = np.arange(n, dtype=np.float32) * np.float32(0.5)
    P[:, 1] = np.arange(n, dtype=np.float32) * np.float32(0.25)
    step = float(ref_dist(metric, P[:1], P[1:2])[0, 0])  # the same for every neighbour pair: the coordinates are exact
    eng = _engine(monkeypatch)
    for perm in (np.arange(n), np.random.default_rng(2).permutation(n)):
        Q = P[perm]
        D = ref_dist(metric, Q, Q)
        for eps in (step * 1.05, step):  # neighbours just under eps, and exactly at it
            labels = _same(eng, Q, metric, eps, 3, D)
            assert (labels == 0).all()
            _same(eng, Q, metric, eps, 2, D)
        labels = _same(eng, Q, metric, float(np.nextafter(np.float32(step), np.float32(0))), 2, D)
        assert (labels == -1).all()  # just below: all noise
    eng.close()


def test_dbscan_all_pairs_in_radius(monkeypatch):
    """A 3,000-point blob with every pair in radius: every union contends for the same root."""
    rng = np.random.default_rng(3)
    P = rng.uniform(-0.5, 0.5, (3000, 28)).astype(np.float32)
    eng = _engine(monkeypatch)
    for metric in METRICS:
        D = ref_dist(metric, P, P)
        labels = _same(eng, P, metric, float(D.max()) * 1.01, 5, D)
        assert (labels == 0).all()
        _same(eng, P, metric, float(D.max()), 3000, D)  # every row core, exactly at the largest distance
    eng.close()


@pytest.mark.parametrize("metric", METRICS)
def test_dbscan_repeated_rows(metric, monkeypatch):
    """Rows drawn from 20 distinct ones: distance-0 ties; eps below every nonzero distance, and at an attained one."""
    rng = np.random.default_rng(7)
    base = rng.choice(np.array([-0.5, 0.0, 0.5], np.float32), (20, 28))
    P = base[rng.integers(0, 20, 1000)]
    D = ref_dist(metric, P, P)
    nz = np.unique(D[D > 0])
    eng = _engine(monkeypatch, 256)
    for eps in (float(nz[0]) / 2, float(nz[0]), float(nz[len(nz) // 3])):
        for ms in (1, 30, 60, 200):
            _same(eng, P, metric, eps, ms, D)
    eng.close()


def test_dbscan_border_rules(monkeypatch):
    """A border row adjacent to two clusters whose nearer one has the larger seed takes the smaller seed's cluster, and
    a border row whose index is below its cluster's seed; as in tests/test_cluster_host.py, on the device."""
    eng = _engine(monkeypatch)
    for x, ms, want in (([-0.9, -1.5, -1.6, -1.8, 0.5, 1.1, 1.2, 1.4, 0.0], 4, [0, 0, 0, 0, 1, 1, 1, 1, 0]),
                        ([3.0, 0.0, 0.5, 1.0, 1.5, 2.0], 4, [0] * 6)):
        P = np.zeros((len(x), 4), np.float32)
        P[:, 0] = x
        for metric in METRICS:
            labels = _same(eng, P, metric, 1.0, ms)
            assert list(labels) == want
    eng.close()


def test_dbscan_deterministic(monkeypatch):
    rng = np.random.default_rng(5)
    P = _dev(_blobs(rng, 4000, 28, centers=30, sigma=0.08))
    eng = _engine(monkeypatch)
    a = eng.dbscan(P, 0.4, 4, "euclidean")
    b = eng.dbscan(P, 0.4, 4, "euclidean")
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and int(a[0].max()) > 5
    eng.close()


def test_dbscan_errors(monkeypatch):
    eng = _engine(monkeypatch)
    P = _dev(np.zeros((10, 4), np.float32))
    with pytest.raises(ValueError, match="eps"):
        eng.dbscan(P, 0.0, 2, "euclidean")
    with pytest.raises(ValueError, match="min_samples"):
        eng.dbscan(P, 0.5, 0, "euclidean")
    with pytest.raises(ValueError, match="unknown metric"):
        eng.dbscan(P, 0.5, 2, "cosine")
    labels, core = eng.dbscan(P[:0], 0.5, 2, "euclidean")
    assert labels.numel() == 0 and core.numel() == 0
    labels, core = eng.dbscan(P, 0.5, 2, "manhattan")
    assert (labels.cpu() == 0).all() and core.all()
    eng.close()


def test_dbscan_scale(monkeypatch):
    """100,000 x 400 clustered points against sklearn's dbscan_inner, applied to the core flags and neighbourhoods of
    kge_radius_neighbors' CSR (bit-exact-tested in tests/test_gpu_knn.py): an n^2 CPU oracle is too slow here."""
    from sklearn.cluster._dbscan_inner import dbscan_inner
    n, ld, ms = 100_000, 400, 10
    g = torch.Generator(device="cuda").manual_seed(9)
    centers = torch.rand((1000, ld), generator=g, device="cuda") - 0.5
    pts = centers[torch.randint(0, 1000, (n,), generator=g, device="cuda")]
    pts += 0.035 * torch.randn((n, ld), generator=g, device="cuda")
    far = torch.rand(n, generator=g, device="cuda") < 0.05
    pts[far] = torch.rand((int(far.sum()), ld), generator=g, device="cuda") - 0.5
    pts = pts.contiguous()
    eng = _engine(monkeypatch)
    for metric, eps in (("euclidean", 1.0), ("manhattan", 16.0)):
        labels, core = (x.cpu().numpy() for x in eng.dbscan(pts, eps, ms, metric))
        every = torch.arange(n, dtype=torch.int32, device="cuda")
        neighborhoods = np.empty(n, dtype=object)
        for s in range(0, n, 8192):
            off, nbr = (x.cpu().numpy() for x in eng.radius_neighbors(pts, every[s:s + 8192], eps, metric))
            for i, row in enumerate(np.split(nbr.astype(np.intp), off[1:-1])):
                neighborhoods[s + i] = row
        counts = np.array([len(r) for r in neighborhoods])
        want_core = counts >= ms
        want = np.full(n, -1, dtype=np.intp)
        dbscan_inner(want_core.astype(np.uint8), neighborhoods, want)
        assert (core == want_core).all()
        assert (labels == want).all(), np.flatnonzero(labels != want)[:5]
        assert want_core.any() and (~want_core).any() and want.max() > 100 and (want == -1).any(), metric
    eng.close()


# ---------------------------------------------------------------------------
def _kg(E, R, n, seed):
    rng = np.random.default_rng(seed)
    t = np.unique(np.stack([rng.integers(0, E, n), rng.integers(0, R, n), rng.integers(0, E, n)], 1), axis=0)
    return np.stack([np.char.add("e", t[:, 0].astype(str)), np.char.add("r", t[:, 1].astype(str)),
                     np.char.add("e", t[:, 2].astype(str))], 1)


@pytest.fixture(scope="module")
def fitted():
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    X = _kg(120, 8, 900, 23)
    m = ScoringBasedEmbeddingModel(eta=3, k=18, scoring_type="ComplEx", seed=4)  # k = 18: padded rows (kp = 20)
    m.compile(optimizer="adam", loss="pairwise")
    m.fit(X, batch_size=150, epochs=3, verbose=False)
    return m, X


def _emb(X, m, mode):
    if mode == "t":
        return np.hstack((m.get_embeddings(X[:, 0], "e"), m.get_embeddings(X[:, 1], "r"), m.get_embeddings(X[:, 2], "e")))
    return m.get_embeddings(X, embedding_type=mode)


def _gap_eps(emb, metric, q):
    """An eps near the q-quantile of the pairwise fp64 distances, in the middle of a gap wider than 1e-4 relative: sklearn
    computes euclidean distances through a GEMM, which may put a pair at the boundary on the other side."""
    from scipy.spatial.distance import pdist
    d = np.unique(pdist(emb.astype(np.float64), "euclidean" if metric == "euclidean" else "cityblock"))
    i = int(q * (len(d) - 1))
    while i + 1 < len(d) and d[i + 1] - d[i] <= 1e-4 * d[i + 1]:
        i += 1
    return float(d[i] + d[i + 1]) / 2


def test_find_clusters_reference_cases():
    """The reference's test_find_clusters (tests/ampligraph/discovery/test_discovery.py:140-178), restated."""
    from sklearn.cluster import DBSCAN
    from ampligraph_b200.discovery import find_clusters
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    X = np.array([['a', 'y', 'b'], ['b', 'y', 'a'], ['a', 'y', 'c'], ['c', 'y', 'a'], ['a', 'y', 'd'], ['c', 'x', 'd'],
                  ['b', 'y', 'c'], ['f', 'y', 'e']])
    model = ScoringBasedEmbeddingModel(eta=5, k=10, scoring_type='ComplEx', seed=0)
    model.compile(optimizer='adam', loss='multiclass_nll')
    model.fit(X, batch_size=1, epochs=10, verbose=False)
    clustering_algorithm = DBSCAN(eps=1e-3, min_samples=1)
    assert np.array_equal(find_clusters(X, model, clustering_algorithm, mode='t'), np.arange(8))
    assert np.array_equal(find_clusters(np.unique(X[:, 0]), model, clustering_algorithm, mode='e'), np.arange(4))
    assert np.array_equal(find_clusters(np.unique(X[:, 1]), model, clustering_algorithm, mode='r'), np.arange(2))
    assert np.array_equal(find_clusters(np.unique(X[:, 2]), model, clustering_algorithm, mode='e'), np.arange(5))
    with pytest.raises(ValueError):
        find_clusters(X, model, clustering_algorithm, mode='hah')
    with pytest.raises(ValueError):
        find_clusters(X, model, clustering_algorithm, mode='e')
    with pytest.raises(ValueError):
        find_clusters(X, model, clustering_algorithm, mode='r')
    with pytest.raises(ValueError):
        find_clusters(np.unique(X[:, 0]), model, clustering_algorithm, mode='t')


@pytest.mark.parametrize("mode", ["e", "r", "t"])
@pytest.mark.parametrize("metric", ["euclidean", "manhattan", "minkowski"])
def test_find_clusters_vs_sklearn(fitted, mode, metric):
    from sklearn.cluster import DBSCAN
    from ampligraph_b200.discovery import find_clusters
    m, X = fitted
    Xm = {"e": np.unique(np.concatenate([X[:, 0], X[:, 2]])), "r": np.unique(X[:, 1]), "t": X[:300]}[mode]
    emb = _emb(Xm, m, mode)
    p = 1 if metric == "minkowski" else None
    for q, ms in ((0.02, 3), (0.1, 5), (0.3, 2)):
        eps = _gap_eps(emb, "manhattan" if metric != "euclidean" else metric, q)
        ref = DBSCAN(eps=eps, min_samples=ms, metric=metric, p=p).fit(emb)
        est = DBSCAN(eps=eps, min_samples=ms, metric=metric, p=p)
        labels = find_clusters(Xm, m, est, mode=mode)
        assert labels.dtype == np.int64 and (labels == ref.labels_).all(), (q, ms)
        assert (est.labels_ == ref.labels_).all()
        assert np.array_equal(est.core_sample_indices_, ref.core_sample_indices_)
        assert est.components_.shape == ref.components_.shape and np.array_equal(est.components_, ref.components_)
        assert est.n_features_in_ == ref.n_features_in_ == emb.shape[1]


def test_find_clusters_host_algorithms(fitted):
    """KMeans (the reference docstring's example), a cosine DBSCAN and a DBSCAN subclass run their own fit_predict."""
    from sklearn.cluster import DBSCAN, KMeans
    from ampligraph_b200.discovery import find_clusters

    class Sub(DBSCAN):
        pass

    m, X = fitted
    ents = np.unique(X[:, 0])
    emb = _emb(ents, m, "e")
    assert (find_clusters(ents, m, KMeans(n_clusters=4, random_state=0, n_init=3)) ==
            KMeans(n_clusters=4, random_state=0, n_init=3).fit_predict(emb)).all()
    assert (find_clusters(ents, m, DBSCAN(eps=0.2, min_samples=2, metric="cosine")) ==
            DBSCAN(eps=0.2, min_samples=2, metric="cosine").fit_predict(emb)).all()
    eps = _gap_eps(emb, "euclidean", 0.05)
    assert (find_clusters(ents, m, Sub(eps=eps, min_samples=2)) == DBSCAN(eps=eps, min_samples=2).fit_predict(emb)).all()


def test_find_clusters_default(fitted):
    """None means DBSCAN()'s defaults: the same labels as DBSCAN() itself."""
    from sklearn.cluster import DBSCAN
    from scipy.spatial.distance import pdist
    from ampligraph_b200.discovery import find_clusters
    m, X = fitted
    ents = np.unique(np.concatenate([X[:, 0], X[:, 2]]))
    emb = _emb(ents, m, "e")
    got = find_clusters(ents, m)
    assert np.array_equal(got, find_clusters(ents, m, DBSCAN()))
    d = pdist(emb.astype(np.float64))
    if not (np.abs(d - 0.5) <= 1e-4).any():  # no pair at the boundary: sklearn's GEMM distances agree
        assert np.array_equal(got, DBSCAN().fit_predict(emb))
    saved = m.engine.ent.clone()
    m.engine.ent *= 0.02  # shrink the table so that the default eps makes a cluster
    try:
        emb = _emb(ents, m, "e")
        got = find_clusters(ents, m)
        d = pdist(emb.astype(np.float64))
        assert not (np.abs(d - 0.5) <= 1e-4).any()
        assert np.array_equal(got, DBSCAN().fit_predict(emb)) and got.max() >= 0
    finally:
        m.engine.ent.copy_(saved)


def test_find_clusters_errors(fitted):
    from sklearn.cluster import DBSCAN
    from ampligraph_b200.discovery import find_clusters
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    m, X = fitted
    ents = np.unique(X[:, 0])
    with pytest.raises(ValueError, match="fit_predict"):
        find_clusters(ents, m, object())
    with pytest.raises(ValueError, match="not been fitted"):
        find_clusters(ents, ScoringBasedEmbeddingModel(eta=1, k=4, scoring_type="TransE"))
    with pytest.raises(ValueError, match="not been seen"):
        find_clusters(np.array(["nope"] + list(ents)), m)
    with pytest.raises(ValueError, match="eps"):
        find_clusters(ents, m, DBSCAN(eps=-1.0))
