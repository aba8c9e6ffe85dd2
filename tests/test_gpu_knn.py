"""GPU tests of nearest-neighbour and radius search: kge_knn / kge_radius_neighbors (csrc/kge_knn.cu with the ranking
pair and tile kernels) through the engine, and the discovery facade (find_nearest_neighbours, find_duplicates).
Ids and distances must equal the ordering contract (tests/topk_oracle.py) applied to the C restatement of the
distance chains (tests/knn_oracle.c), bit for bit."""
import logging

import numpy as np
import pytest
import torch

from knn_oracle import distances as ref_dist
from topk_oracle import topk as ref_topk

pytestmark = pytest.mark.gpu

METRICS = ["euclidean", "manhattan"]


def _dev(a):
    return torch.as_tensor(a).cuda().contiguous()


def _engine(monkeypatch, chunk=None):
    from ampligraph_b200.engine import KGEEngine
    if chunk is None:
        monkeypatch.delenv("KGE_B200_TOPK_CHUNK", raising=False)
    else:
        monkeypatch.setenv("KGE_B200_TOPK_CHUNK", str(chunk))  # read when the handle is created
    return KGEEngine("TransE", 4, 1, 8, 1)  # the handle only lends its device and chunk rule to kge_knn


def _expect(D, k, farthest=False, exclude=None, to_id=None):
    """ids / distances kge_knn must return for the candidate distance matrix D [b, n_cand]."""
    pos, val = ref_topk(D if farthest else -D, k, exclude)
    ids = pos if to_id is None else np.where(pos >= 0, to_id(np.maximum(pos, 0)), -1)
    return ids, (val if farthest else -val)


def _same(got, want):
    gi, gd = (x.cpu().numpy() for x in got)
    wi, wd = want
    assert gi.shape == wi.shape and (gi == wi).all(), np.argwhere(gi != wi)[:5]
    assert (gd.view(np.uint32) == wd.astype(np.float32).view(np.uint32)).all(), np.argwhere(gd != wd)[:5]


# ---------------------------------------------------------------------------
@pytest.mark.parametrize("kernel", ["pair", "tile"])
@pytest.mark.parametrize("chunk", [None, 256])
@pytest.mark.parametrize("metric", METRICS)
def test_knn_vs_oracle(metric, chunk, kernel, monkeypatch):
    """Widths 4, 28 (a column-chunk tail), 400 and 1,200 (a triple's width); all candidates, a window and an unsorted
    cand_ids subset; k = 1, 7, n_cand and beyond n_cand (padding); nearest and farthest."""
    if kernel == "tile":
        monkeypatch.setenv("KGE_B200_RANK_KERNEL", "tile")
    else:
        monkeypatch.delenv("KGE_B200_RANK_KERNEL", raising=False)
    rng = np.random.default_rng(31)
    n, b = 700, 37
    eng = _engine(monkeypatch, chunk)
    sub = rng.choice(n, 300, replace=False).astype(np.int32)
    qids = rng.integers(0, n, b).astype(np.int32)
    for ld in (4, 28, 400, 1200):
        P = rng.uniform(-0.5, 0.5, (n, ld)).astype(np.float32)
        D = ref_dist(metric, P[qids], P)
        pts, q = _dev(P), _dev(qids)
        for far in (False, True):
            for top in (1, 7, 300, 305):
                _same(eng.knn(pts, q, top, metric, farthest=far), _expect(D, top, far))
                _same(eng.knn(pts, q, top, metric, cand_begin=250, n_cand=300, farthest=far),
                      _expect(D[:, 250:550], top, far, to_id=lambda p: p + 250))
                _same(eng.knn(pts, q, top, metric, cand_ids=_dev(sub), farthest=far),
                      _expect(D[:, sub], top, far, to_id=lambda p: sub[p]))
            _same(eng.knn(pts, q, n, metric, farthest=far), _expect(D, n, far))
    eng.close()


@pytest.mark.parametrize("metric", METRICS)
def test_knn_ties_and_self_exclusion(metric, monkeypatch):
    """Rows drawn from 20 distinct ones: many equal distances, zeros among them, ordered by position whatever the chunk;
    excluding each query's own position returns its nearest OTHER row (distance 0 for a repeated row)."""
    rng = np.random.default_rng(7)
    n, ld = 1000, 28
    base = rng.choice(np.array([-0.5, 0.0, 0.5], np.float32), (20, ld))
    P = base[rng.integers(0, 20, n)]
    qids = np.arange(n, dtype=np.int32)
    D = ref_dist(metric, P, P)
    off = np.arange(n + 1, dtype=np.int64)
    for chunk in (None, 256, 100):
        eng = _engine(monkeypatch, chunk)
        pts, q = _dev(P), _dev(qids)
        _same(eng.knn(pts, q, 60, metric), _expect(D, 60))
        got = eng.knn(pts, q, 3, metric, filt_off=_dev(off), filt_idx=q)
        _same(got, _expect(D, 3, exclude=[[i] for i in range(n)]))
        ids = got[0].cpu().numpy()
        assert (ids[:, 0] != qids).all()
        eng.close()


def _radius_ref(D, r):
    rows = [np.nonzero(D[i] <= np.float32(r))[0] for i in range(len(D))]
    off = np.concatenate([[0], np.cumsum([len(x) for x in rows])]).astype(np.int64)
    return off, (np.concatenate(rows) if off[-1] else np.zeros(0, np.int64))


@pytest.mark.parametrize("chunk", [None, 256])
@pytest.mark.parametrize("metric", METRICS)
def test_radius_vs_oracle(metric, chunk, monkeypatch):
    """r = 0, r equal to an attained distance (inclusive), r above every distance; a window and a subset; and the
    consistency find_duplicates rests on: rows with more than one neighbour are exactly {i : d1(i) <= r}."""
    rng = np.random.default_rng(3)
    n, ld = 900, 28
    base = rng.uniform(-0.5, 0.5, (300, ld)).astype(np.float32)
    P = base[rng.integers(0, 300, n)]  # repeated rows: zero distances between different positions
    D = ref_dist(metric, P, P)
    eng = _engine(monkeypatch, chunk)
    pts, q = _dev(P), _dev(np.arange(n, dtype=np.int32))
    off = np.arange(n + 1, dtype=np.int64)
    d1 = eng.knn(pts, q, 1, metric, filt_off=_dev(off), filt_idx=q)[1].cpu().numpy()[:, 0]
    radii = [-1.0, 0.0, float(D[0, 5]), float(D[17, 400]), float(np.median(d1)), float(D.max()) + 1.0]
    for r in radii:
        o, ids = (x.cpu().numpy() for x in eng.radius_neighbors(pts, q, r, metric))
        wo, wids = _radius_ref(D, r)
        assert (o == wo).all() and (ids == wids).all(), r
        assert set(np.nonzero(np.diff(o) > 1)[0]) == set(np.nonzero(d1 <= np.float32(r))[0])
    r = float(D[3, 9])
    sub = rng.choice(n, 250, replace=False).astype(np.int32)
    o, ids = (x.cpu().numpy() for x in eng.radius_neighbors(pts, q[:50], r, metric, cand_ids=_dev(sub)))
    wo, wpos = _radius_ref(D[:50][:, sub], r)
    assert (o == wo).all() and (ids == sub[wpos]).all()
    o, ids = (x.cpu().numpy() for x in eng.radius_neighbors(pts, q[:50], r, metric, cand_begin=100, n_cand=600))
    wo, wpos = _radius_ref(D[:50, 100:700], r)
    assert (o == wo).all() and (ids == wpos + 100).all()
    eng.close()


def test_knn_scale_cfg2(monkeypatch):
    """The cfg2-sized self-join (14,505 x 400, every row a query, top 10), 64 sampled rows against the oracle."""
    rng = np.random.default_rng(17)
    n, ld = 14505, 400
    P = rng.uniform(-0.5, 0.5, (n, ld)).astype(np.float32)
    eng = _engine(monkeypatch)
    pts = _dev(P)
    sample = rng.choice(n, 64, replace=False)
    for metric in METRICS:
        ids, d = eng.knn(pts, _dev(np.arange(n, dtype=np.int32)), 10, metric)
        _same((ids[sample], d[sample]), _expect(ref_dist(metric, P[sample], P), 10))
    eng.close()


def test_knn_million_points(monkeypatch):
    """16 queries against 1,000,000 rows of 400 floats (1.6 GB, many L2-sized chunks).  The oracle's exact chain runs
    only on the candidates a float64 pre-pass puts near the 50-th distance; the margin covers its rounding many times."""
    n, ld, b, top = 1_000_000, 400, 16, 50
    g = torch.Generator(device="cuda").manual_seed(5)
    pts = torch.rand((n, ld), generator=g, device="cuda", dtype=torch.float32) - 0.5
    qids = torch.randint(0, n, (b,), generator=g, device="cuda", dtype=torch.int32)
    eng = _engine(monkeypatch)
    ids, d = (x.cpu().numpy() for x in eng.knn(pts, qids, top, "euclidean"))
    Q = pts[qids.long()].double()
    d2 = torch.cat([((Q[:, None, :] - pts[None, c0:c0 + 20_000].double()) ** 2).sum(-1) for c0 in range(0, n, 20_000)], 1)
    kth = torch.kthvalue(d2, top, dim=1).values
    for i in range(b):
        near = torch.nonzero(d2[i] <= kth[i] * (1 + 1e-3)).flatten()  # ascending positions: ties keep their order
        rows = pts[near].cpu().numpy()
        q = pts[qids[i].long()].cpu().numpy()[None]
        wpos, wd = _expect(ref_dist("euclidean", q, rows), top)
        assert (ids[i] == near.cpu().numpy()[wpos[0]]).all(), i
        assert (d[i].view(np.uint32) == wd[0].view(np.uint32)).all(), i
    eng.close()


def test_knn_errors(monkeypatch):
    import ctypes as C
    from ampligraph_b200 import _lib
    from ampligraph_b200.engine import _ptr
    eng = _engine(monkeypatch)
    pts = _dev(np.zeros((50, 8), np.float32))
    q = _dev(np.array([1, 2], np.int32))
    with pytest.raises(ValueError, match="k must be"):
        eng.knn(pts, q, 0, "euclidean")
    with pytest.raises(ValueError, match="unknown metric"):
        eng.knn(pts, q, 3, "cosine")
    with pytest.raises(ValueError, match="exceeds n_points"):
        eng.knn(pts, q, 3, "euclidean", cand_begin=10, n_cand=45)
    with pytest.raises(ValueError, match="multiple of 4"):
        eng.knn(_dev(np.zeros((50, 6), np.float32)), q, 3, "euclidean")
    with pytest.raises(ValueError, match="16-byte aligned"):
        eng.knn(torch.zeros(50 * 8 + 1, device="cuda")[1:].view(50, 8), q, 3, "euclidean")
    with pytest.raises(ValueError, match="exceeds n_points"):
        eng.radius_neighbors(pts, q, 0.5, "manhattan", cand_begin=49, n_cand=2)
    lib = eng.lib
    need = lib.kge_knn_workspace_bytes(eng.h, 2, 50, 3, 8)
    raw = torch.empty(need + 4096, dtype=torch.uint8, device="cuda")
    base = raw.data_ptr() + (-raw.data_ptr()) % 1024
    ids = torch.empty((2, 3), dtype=torch.int32, device="cuda")
    dist = torch.empty((2, 3), dtype=torch.float32, device="cuda")

    def call(ws, nbytes, filt_off=None, n_filt=0):
        return lib.kge_knn(eng.h, 0, _ptr(pts), 50, 8, _ptr(q), 2, None, 0, 50, _ptr(filt_off), None, n_filt, 3, 0,
                           _ptr(ids), _ptr(dist), C.c_void_p(ws), nbytes, eng._stream())
    with pytest.raises(ValueError, match="workspace of"):
        _lib.check(call(base, need - 1))
    with pytest.raises(ValueError, match="aligned"):
        _lib.check(call(base + 256, need))
    with pytest.raises(ValueError, match="given together"):
        _lib.check(call(base, need, _dev(np.zeros(3, np.int64)), 2))
    _lib.check(call(base, need))
    assert lib.kge_knn(eng.h, 0, None, 0, 8, None, 0, None, 0, 0, None, None, 0, 3, 0, None, None, None, 0, None) == 0
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


@pytest.mark.parametrize("metric,sk_metric", [("euclidean", "euclidean"), ("l1", "manhattan")])
def test_find_nearest_neighbours_vs_sklearn(fitted, metric, sk_metric):
    from sklearn.neighbors import NearestNeighbors
    from ampligraph_b200.discovery import find_nearest_neighbours
    m, X = fitted
    labels = np.array(sorted(set(X[:, 0]) | set(X[:, 2])))
    ents = list(labels[::7])
    for subset in (None, list(labels[5:90][::-1])):
        cand = subset if subset is not None else list(m.data_indexer.ent_labels)
        emb = m.get_embeddings(np.array(cand))
        dist, idx = NearestNeighbors(n_neighbors=6, metric=sk_metric).fit(emb).kneighbors(m.get_embeddings(np.array(ents)))
        got, gd = find_nearest_neighbours(m, ents, n_neighbors=6, entities_subset=subset, metric=metric)
        assert got.shape == (len(ents), 6) and gd.shape == (len(ents), 6) and gd.dtype == np.float32
        assert (got == np.asarray(cand)[idx]).all()
        np.testing.assert_allclose(gd, dist, rtol=1e-5, atol=1e-6)  # sklearn: |x|^2 + |y|^2 - 2xy, not 0 at x = y


def _emb(X, m, mode):
    if mode == "t":
        return np.hstack((m.get_embeddings(X[:, 0], "e"), m.get_embeddings(X[:, 1], "r"), m.get_embeddings(X[:, 2], "e")))
    return m.get_embeddings(X, embedding_type=mode)


def _reference_duplicates(X, m, mode, metric, tolerance, expected=0.1):
    """discovery.py:914-982, restated with sklearn / scipy on the model's dense embeddings."""
    from scipy import optimize, spatial
    from sklearn.neighbors import NearestNeighbors
    emb = _emb(X, m, mode)

    def get_dups(tol):
        nn = NearestNeighbors(metric=metric, radius=tol)
        nn.fit(emb)
        neighbors = nn.radius_neighbors(emb)[1]
        idx_dups = ((i, row) for i, row in enumerate(neighbors) if len(row) > 1)
        if mode == "t":
            return {frozenset(tuple(X[idx]) for idx in row) for i, row in idx_dups}
        return {frozenset(X[idx] for idx in row) for i, row in idx_dups}

    def opt(tol, info):
        return len(set().union(*get_dups(tol))) / len(emb) - expected

    if tolerance == "auto":
        max_distance = spatial.distance_matrix(emb, emb).max()
        tolerance = optimize.bisect(opt, 0.0, max_distance, xtol=1e-3, maxiter=50, args=({"Nfeval": 0},))
    return get_dups(tolerance), tolerance


@pytest.mark.parametrize("mode", ["e", "r", "t"])
@pytest.mark.parametrize("metric", ["l2", "manhattan"])
def test_find_duplicates_vs_reference(fitted, mode, metric):
    from sklearn.neighbors import NearestNeighbors
    from ampligraph_b200.discovery import find_duplicates
    m, X = fitted
    if mode == "e":
        Xm = np.concatenate([np.unique(X[:, 0]), X[:5, 0]])  # repeated labels
    elif mode == "r":
        Xm = np.unique(X[:, 1])
    else:
        Xm = np.concatenate([X[:200], X[:3]])
    sk = "euclidean" if metric == "l2" else metric
    if metric == "l2":
        ref_dups, ref_tol = _reference_duplicates(Xm, m, mode, sk, "auto")
        dups, got_tol = find_duplicates(Xm, m, mode=mode, metric=metric)
        assert abs(got_tol - ref_tol) <= 1e-3
        assert dups == ref_dups and len(dups) > 0
    else:
        # the bracket ends at the largest EUCLIDEAN distance (:972); manhattan distances are longer, so the fraction there
        # stays below the expected one and the reference's bisect refuses the bracket -- and so does find_duplicates
        with pytest.raises(ValueError, match="different signs"):
            _reference_duplicates(Xm, m, mode, sk, "auto")
        with pytest.raises(ValueError, match="different signs"):
            find_duplicates(Xm, m, mode=mode, metric=metric)
    # an explicit tolerance halfway between two attained nearest-other distances
    emb = _emb(Xm, m, mode)
    d1 = np.unique(NearestNeighbors(n_neighbors=2, metric=sk).fit(emb).kneighbors(emb)[0][:, 1])
    tol = float(d1[len(d1) // 2] + d1[len(d1) // 2 + 1]) / 2
    dups, got_tol = find_duplicates(Xm, m, mode=mode, metric=metric, tolerance=tol)
    assert got_tol == tol and dups == _reference_duplicates(Xm, m, mode, sk, tol)[0] and len(dups) > 0


def test_find_duplicates_auto_verbose(fitted, caplog):
    from ampligraph_b200.discovery import find_duplicates
    m, X = fitted
    with caplog.at_level(logging.INFO, logger="ampligraph_b200.discovery"):
        find_duplicates(np.unique(X[:, 0]), m, tolerance="auto", verbose=True)
    assert any("Eval 1: tol:" in r.message for r in caplog.records)


def test_knn_facade_errors(fitted):
    from ampligraph_b200.discovery import find_duplicates, find_nearest_neighbours
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    m, X = fitted
    ents = np.unique(X[:, 0])
    with pytest.raises(ValueError, match="`mode` must be one of"):
        find_duplicates(ents, m, mode="x")
    with pytest.raises(ValueError, match="three columns"):
        find_duplicates(ents, m, mode="t")
    with pytest.raises(ValueError, match="must be an array"):
        find_duplicates(X, m, mode="e")
    with pytest.raises(ValueError, match="must be an array"):
        find_duplicates(X[:, :2], m, mode="r")
    unfitted = ScoringBasedEmbeddingModel(eta=1, k=4, scoring_type="TransE")
    with pytest.raises(ValueError, match="not been fitted"):
        find_duplicates(ents, unfitted)
    with pytest.raises(AssertionError, match="not fit"):
        find_nearest_neighbours(unfitted, list(ents[:2]))
    with pytest.raises(AssertionError, match="Invalid type for entities!"):
        find_nearest_neighbours(m, "e1")
    with pytest.raises(AssertionError, match="Invalid type for entities_subset"):
        find_nearest_neighbours(m, list(ents[:2]), entities_subset="e1")
    with pytest.raises(AssertionError, match="n_neighbors must be less"):
        find_nearest_neighbours(m, list(ents[:2]), n_neighbors=5, entities_subset=list(ents[:5]))
    for bad in ("cosine", "chebyshev", lambda a, b: 0.0):
        with pytest.raises(NotImplementedError, match="supported"):
            find_nearest_neighbours(m, list(ents[:2]), metric=bad)
        with pytest.raises(NotImplementedError, match="supported"):
            find_duplicates(ents, m, metric=bad, tolerance=0.1)


def test_knn_facade_non_finite():
    from ampligraph_b200.discovery import find_duplicates, find_nearest_neighbours
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    X = _kg(30, 3, 120, 9)
    m = ScoringBasedEmbeddingModel(eta=2, k=8, scoring_type="DistMult", seed=1)
    m.compile(optimizer="adam", loss="pairwise")
    m.fit(X, batch_size=60, epochs=1, verbose=False)
    ents = np.unique(X[:, 0])
    i = m.get_indexes(np.array([ents[1]]), "e")[0]
    m.engine.ent[i, 0] = float("nan")
    with pytest.raises(ValueError, match="NaN or infinity"):
        find_nearest_neighbours(m, list(ents[:3]), n_neighbors=2)
    with pytest.raises(ValueError, match="NaN or infinity"):
        find_duplicates(ents, m, tolerance=0.5)
    m.engine.ent[i, 0] = float("inf")
    with pytest.raises(ValueError, match="NaN or infinity"):
        find_duplicates(ents, m, tolerance="auto")


def test_find_duplicates_manhattan_auto_vs_reference():
    """A manhattan bisection that converges: 12 pairs of near-duplicate entities at manhattan distances 0.05 .. 0.6, far
    inside the bracket [0, largest euclidean distance], so the duplicate fraction crosses the expected one there."""
    from ampligraph_b200.discovery import find_duplicates
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    X = _kg(60, 3, 300, 13)
    m = ScoringBasedEmbeddingModel(eta=2, k=8, scoring_type="DistMult", seed=2)
    m.compile(optimizer="adam", loss="pairwise")
    m.fit(X, batch_size=100, epochs=1, verbose=False)
    ents = np.unique(np.concatenate([X[:, 0], X[:, 2]]))
    ids = m.get_indexes(ents, "e")
    rng = np.random.default_rng(8)
    ent = rng.uniform(-1, 1, (m.engine.n_ent, 8)).astype(np.float32)
    for j, r in enumerate(np.linspace(0.05, 0.6, 12)):
        ent[ids[2 * j + 1]] = ent[ids[2 * j]] + np.float32(r / 8) * np.sign(rng.standard_normal(8)).astype(np.float32)
    m.engine.set_embeddings(ent, m.engine.get_embeddings()[1])
    ref_dups, ref_tol = _reference_duplicates(ents, m, "e", "manhattan", "auto", expected=0.15)
    dups, tol = find_duplicates(ents, m, metric="manhattan", expected_fraction_duplicates=0.15)
    assert 0.0 < ref_tol < 0.6
    assert abs(tol - ref_tol) <= 1e-3
    assert dups == ref_dups and len(dups) >= 4
