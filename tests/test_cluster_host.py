"""CPU tests of the DBSCAN plumbing: the relabelling rule dbscan_labels (the O(n) step after the device's union-find)
against sklearn's DBSCAN, and the routing of find_clusters between the GPU and the host."""
import numpy as np
import pytest
import torch
from scipy.sparse import csgraph
from scipy.spatial.distance import cdist
from sklearn.cluster import DBSCAN, KMeans

from ampligraph_b200.discovery import _dbscan_on_gpu
from ampligraph_b200.engine import INT32_MAX, dbscan_labels


def _union_find_result(D, eps, min_samples):
    """What the device computes, from scipy: core flags, each core row's smallest component member (the root of its
    union-find tree) and each non-core row's smallest root among its core neighbours (INT32_MAX: none)."""
    A = D <= eps
    core = A.sum(1) >= min_samples
    n = len(D)
    root = np.arange(n)
    core_ids = np.flatnonzero(core)
    if len(core_ids):
        _, comp = csgraph.connected_components(A[np.ix_(core_ids, core_ids)], directed=False)
        seed = np.full(comp.max() + 1, n)
        np.minimum.at(seed, comp, core_ids)
        root[core_ids] = seed[comp]
    border = np.full(n, INT32_MAX, np.int64)
    for i in np.flatnonzero(~core):
        nb = core_ids[A[i, core_ids]]
        if len(nb):
            border[i] = root[nb].min()
    return core, root, border


def _check(P, eps, min_samples):
    D = cdist(P, P).astype(np.float64)
    want = DBSCAN(eps=eps, min_samples=min_samples, metric="precomputed").fit_predict(D)
    core, root, border = _union_find_result(D, eps, min_samples)
    got = dbscan_labels(torch.as_tensor(core), torch.as_tensor(root, dtype=torch.int32),
                        torch.as_tensor(border, dtype=torch.int32))
    assert got.dtype == torch.int64
    assert (got.numpy() == want).all(), (eps, min_samples, got.numpy(), want)
    return want


def test_dbscan_labels_random_integer_sets():
    """Random integer point sets, eps at quantiles of D and equal to attained distances (ties exactly at eps), repeated
    rows, min_samples from 1 to beyond n."""
    rng = np.random.default_rng(0)
    kinds = set()
    for trial in range(150):
        n = int(rng.integers(1, 60))
        P = rng.integers(0, int(rng.integers(2, 8)), (n, int(rng.integers(1, 4)))).astype(np.float64)
        D = cdist(P, P)
        eps_list = [float(rng.choice(D.ravel())) or 0.5, float(np.quantile(D, 0.1)) + 0.25, 0.5]
        for eps in eps_list:
            for ms in (1, 2, 3, 5, 7, n + 1):
                want = _check(P, eps, ms)
                kinds.add("noise" if (want == -1).all() else "one" if (want == 0).all() else "mixed")
    assert kinds == {"noise", "one", "mixed"}


def test_dbscan_labels_edge_sets():
    rng = np.random.default_rng(1)
    P = rng.integers(0, 3, (40, 2)).astype(np.float64)  # many repeated rows: distance-0 ties
    for ms in (1, 2, 4, 9, 41):
        _check(P, 1.0, ms)
    _check(np.arange(20, dtype=np.float64)[:, None] * 10, 1.0, 2)  # all noise
    _check(np.arange(20, dtype=np.float64)[:, None], 1.0, 2)  # one chain, one component
    _check(rng.uniform(0, 1, (30, 3)), 10.0, 5)  # every pair in radius
    # a border row next to two clusters, the nearer one with the larger seed: the smaller seed wins
    P = np.array([-0.9, -1.5, -1.6, -1.8, 0.5, 1.1, 1.2, 1.4, 0.0])[:, None]
    want = _check(P, 1.0, 4)
    assert list(want) == [0, 0, 0, 0, 1, 1, 1, 1, 0]
    # a border row whose index is below its cluster's seed (row 0 is reached from seed 2)
    P = np.array([3.0, 0.0, 0.5, 1.0, 1.5, 2.0])[:, None]
    want = _check(P, 1.0, 4)
    assert list(want) == [0] * 6 and list(DBSCAN(eps=1.0, min_samples=4).fit(P).core_sample_indices_) == [2, 3, 4, 5]


def test_dbscan_labels_empty():
    e = torch.zeros(0, dtype=torch.int32)
    assert dbscan_labels(torch.zeros(0, dtype=torch.bool), e, e).numel() == 0


class _MyDBSCAN(DBSCAN):
    pass


def test_routing():
    assert _dbscan_on_gpu(None) == (0.5, 5, "euclidean")
    assert _dbscan_on_gpu(DBSCAN()) == (0.5, 5, "euclidean")
    assert _dbscan_on_gpu(DBSCAN(eps=0.2, min_samples=3, metric="minkowski", p=2)) == (0.2, 3, "euclidean")
    assert _dbscan_on_gpu(DBSCAN(metric="minkowski", p=1)) == (0.5, 5, "manhattan")
    assert _dbscan_on_gpu(DBSCAN(metric="minkowski", p=1.0)) == (0.5, 5, "manhattan")
    assert _dbscan_on_gpu(DBSCAN(metric="euclidean", p=1)) == (0.5, 5, "euclidean")  # p only matters for minkowski
    for metric in ("l2", "l1", "manhattan", "cityblock"):
        assert _dbscan_on_gpu(DBSCAN(metric=metric))[2] == ("euclidean" if metric == "l2" else "manhattan")
    assert _dbscan_on_gpu(DBSCAN(algorithm="brute", leaf_size=3, n_jobs=2)) == (0.5, 5, "euclidean")
    for host in (DBSCAN(metric="minkowski", p=3), DBSCAN(metric="minkowski"), DBSCAN(metric_params={}),
                 DBSCAN(metric="cosine"), DBSCAN(metric="chebyshev"), DBSCAN(metric=lambda a, b: 0.0), _MyDBSCAN(),
                 KMeans(n_clusters=2)):
        assert _dbscan_on_gpu(host) is None, host
