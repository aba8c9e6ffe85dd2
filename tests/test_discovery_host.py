"""generate_candidates, _setdiff2d and the argument checks of discover_facts on the host, against the reference's
outputs (tests/golden/discovery_candidates.json), and the graph-count restatement (tests/graph_oracle.py) against
networkx.  No GPU: the cluster strategies run here with the restatement in place of engine.graph_counts; the GPU
tests run them on the kernel."""
import builtins
import json
import logging
import os
import sys
import types

import networkx as nx
import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import graph_oracle  # noqa: E402
from ampligraph_b200 import discovery, engine  # noqa: E402
from ampligraph_b200.datasets import DataIndexer  # noqa: E402

with open(os.path.join(ROOT, "tests", "golden", "discovery_candidates.json")) as f:
    GOLDEN = json.load(f)
DATASETS = {k: np.array(v) for k, v in GOLDEN["datasets"].items()}
HOST = ("random_uniform", "entity_frequency", "graph_degree")
CLUSTER = ("cluster_coefficient", "cluster_triangles", "cluster_squares")


def _case_id(c):
    return "%s-%s-%s-%s-%s-%s" % (c["dataset"], c["strategy"], c["target_rel"], c["max_candidates"],
                                  int(c["consolidate_sides"]), c["seed"])


def check_case(c):
    X = DATASETS[c["dataset"]]
    kw = {k: c[k] for k in ("strategy", "target_rel", "max_candidates", "consolidate_sides", "seed")}
    if "error" in c:
        with pytest.raises(getattr(builtins, c["error"][0])):
            discovery.generate_candidates(X, **kw)
        return
    out = discovery.generate_candidates(X, **kw)
    want = np.array(c["out"], dtype=object).reshape(-1, 3)
    assert out.dtype == object and out.shape == want.shape
    assert np.array_equal(out, want)


@pytest.mark.parametrize("case", [c for c in GOLDEN["candidates"] if c["strategy"] in HOST], ids=_case_id)
def test_host_strategies_match_reference(case):
    check_case(case)


def _oracle_graph_counts(triples, n_nodes, device=None):
    import torch
    t = np.asarray(triples)
    return {k: torch.as_tensor(v) for k, v in graph_oracle.counts(t[:, 0], t[:, 2], int(n_nodes)).items()}


@pytest.mark.parametrize("case", [c for c in GOLDEN["candidates"] if c["strategy"] in CLUSTER], ids=_case_id)
def test_cluster_weights_on_the_host_restatement(case, monkeypatch):
    """The host half of the cluster strategies (weights from the counts, normalisation, sampling, filter) with the
    restatement standing in for the kernel."""
    monkeypatch.setattr(engine, "graph_counts", _oracle_graph_counts)
    check_case(case)


@pytest.mark.parametrize("i", range(len(GOLDEN["setdiff2d"])))
def test_setdiff2d_matches_reference(i):
    c = GOLDEN["setdiff2d"][i]
    out = discovery._setdiff2d(np.array(c["A"]), np.array(c["B"]))
    assert out.tolist() == c["out"]


def test_setdiff2d_keeps_later_duplicates():
    A = np.array([["a", "y", "b"], ["a", "y", "b"], ["c", "y", "d"]])
    assert discovery._setdiff2d(A, np.array([["a", "y", "b"]])).tolist() == [["a", "y", "b"], ["c", "y", "d"]]
    with pytest.raises(RuntimeError, match="Input arrays must be 2-dimensional."):
        discovery._setdiff2d(A[0], A)


def test_generate_candidates_argument_errors(caplog):
    X = DATASETS["reference_test"]
    with pytest.raises(ValueError, match="error is not a valid candidate generation strategy."):
        discovery.generate_candidates(X, "error", "rel_0", 10)
    with pytest.raises(ValueError, match="Parameter max_candidates must be a float or int."):
        discovery.generate_candidates(X, "random_uniform", "rel_0", "10")
    with pytest.raises(ValueError, match=r"Parameter max_candidates must be a positive integer or float in range"):
        discovery.generate_candidates(X, "random_uniform", "rel_0", 0)
    with caplog.at_level(logging.WARNING, logger="ampligraph_b200.discovery"):
        out = discovery.generate_candidates(X, "random_uniform", "missing", 10)
    assert "Target relation is not found in triples." in caplog.text
    assert len(out) == 10 and (out[:, 1] == "missing").all()
    # 'exhaustive' stays rejected, as in the reference
    with pytest.raises(ValueError, match="exhaustive is not a valid candidate generation strategy."):
        discovery.generate_candidates(X, "exhaustive", "rel_0", 10)


def test_global_rng_untouched():
    np.random.seed(123)
    want = np.random.random_sample()
    np.random.seed(123)
    discovery.generate_candidates(DATASETS["zipf"], "entity_frequency", "r1", 50, seed=4)
    assert np.random.random_sample() == want


def test_discover_facts_argument_errors():
    """The checks of discover_facts that run before any ranking (the reference's test_discover_facts)."""
    X = DATASETS["reference_test"]
    model = types.SimpleNamespace(is_fitted=False, data_indexer=DataIndexer(X))
    with pytest.raises(ValueError, match="Model is not fitted."):
        discovery.discover_facts(X, model)
    model.is_fitted = True
    with pytest.raises(ValueError, match="error is not a valid strategy."):
        discovery.discover_facts(X, model, strategy="error")
    with pytest.raises(ValueError, match="exhaustive is not a valid strategy."):
        discovery.discover_facts(X, model, strategy="exhaustive")
    with pytest.raises(ValueError, match=r"Target relation\(s\) not found in model: \['error'\]"):
        discovery.discover_facts(X, model, strategy="random_uniform", target_rel="error")
    with pytest.raises(ValueError, match="Parameter max_candidates must be a float or int."):
        discovery.discover_facts(X, model, max_candidates="10", target_rel="rel_0")


# -- the restatement against networkx ------------------------------------------------------------------------------

def _networkx(s, o, n):
    G = nx.Graph()
    G.add_nodes_from(range(n))
    for a, b in zip(s.tolist(), o.tolist()):
        G.add_edge(a, b)
    deg = np.array([G.degree[v] for v in range(n)], np.int64)
    tri = nx.triangles(G)
    cl = nx.clustering(G)
    sq = nx.square_clustering(G)
    return (deg, np.array([tri[v] for v in range(n)], np.int64), np.array([cl[v] for v in range(n)], np.float64),
            np.array([sq[v] for v in range(n)], np.float64))


def _random_graph(seed, n, m, loops, repeats):
    rng = np.random.default_rng(seed)
    w = 1.0 / np.arange(1, n + 1) ** 0.8
    p = w / w.sum()
    s, o = rng.choice(n, m, p=p), rng.choice(n, m, p=p)
    s[:loops] = o[:loops]
    idx = rng.integers(0, m, repeats)
    return np.concatenate([s, o[idx]]), np.concatenate([o, s[idx]])  # repeats in both directions


GRAPHS = {
    "random_a": _random_graph(0, 60, 400, 8, 50) + (60,),
    "random_b": _random_graph(1, 200, 900, 20, 100) + (200,),
    "random_sparse": _random_graph(2, 150, 160, 5, 10) + (150,),
    "star": (np.zeros(30, np.int64), np.arange(1, 31), 31),
    "clique": tuple(np.array(e) for e in zip(*[(a, b) for a in range(9) for b in range(9) if a < b])) + (9,),
    "path": (np.arange(20), np.arange(1, 21), 21),
    "isolated": (np.array([0, 3, 3]), np.array([1, 3, 4]), 8),
    "empty": (np.zeros(0, np.int64), np.zeros(0, np.int64), 5),
    "no_nodes": (np.zeros(0, np.int64), np.zeros(0, np.int64), 0),
}


@pytest.mark.parametrize("name", list(GRAPHS))
def test_oracle_equals_networkx(name):
    s, o, n = GRAPHS[name]
    c = graph_oracle.counts(s, o, n, wedges_per_block=97)  # small blocks: the block loop runs many times
    tri, cl, sq = graph_oracle.networkx_stats(c)
    deg_nx, tri_nx, cl_nx, sq_nx = _networkx(s, o, n)
    assert np.array_equal(c["degree"], deg_nx)
    assert np.array_equal(tri, tri_nx)
    assert np.array_equal(cl.view(np.int64), cl_nx.view(np.int64))
    assert np.array_equal(sq.view(np.int64), sq_nx.view(np.int64))


def test_complete_bipartite_closed_form():
    s, o, want = graph_oracle.complete_bipartite_2(40)
    got = graph_oracle.counts(s, o, 42)
    for k in want:
        assert np.array_equal(got[k], want[k]), k
