"""GPU tests of the per-node wedge counts (kge_graph_counts, csrc/kge_graph.cu, through engine.graph_counts) and of
the discovery functions built on them: generate_candidates' cluster strategies and discover_facts.

The counts are integers, so they must equal the restatement (tests/graph_oracle.py) exactly, on both counter paths
(shared memory, and the workspace slices above the shared-memory bound)."""
import logging
import os
import sys

import numpy as np
import pytest
import torch

import graph_oracle
from test_discovery_host import CLUSTER, DATASETS, GOLDEN, _case_id, _networkx, GRAPHS, check_case

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEYS = ("degree", "d", "tri2", "sq", "pot")


def _gpu(s, o, n):
    t = np.stack([np.asarray(s), np.zeros(len(s), np.int64), np.asarray(o)], 1).astype(np.int64)
    from ampligraph_b200.engine import graph_counts
    got = graph_counts(torch.as_tensor(t).cuda(), n)
    assert all(v.dtype == torch.int64 and v.is_cuda and v.numel() == n for v in got.values())
    return {k: v.cpu().numpy() for k, v in got.items()}


def _assert_equal(got, want):
    for k in KEYS:
        assert np.array_equal(got[k], want[k]), (k, np.flatnonzero(got[k] != want[k])[:10])


def _shared_bound():
    """The largest node count whose counters the library keeps in shared memory (its workspace is then only the
    256-byte work counter)."""
    from ampligraph_b200 import _lib
    ws = _lib.load().kge_graph_workspace_bytes
    lo, hi = 1, 1 << 20
    while lo < hi:
        mid = (lo + hi + 1) // 2
        lo, hi = (mid, hi) if ws(mid) == 256 else (lo, mid - 1)
    return lo


@pytest.mark.parametrize("name", list(GRAPHS))
def test_small_graphs_against_networkx(name):
    s, o, n = GRAPHS[name]
    got = _gpu(s, o, n)
    _assert_equal(got, graph_oracle.counts(s, o, n))
    tri, cl, sq = graph_oracle.networkx_stats(got)
    deg_nx, tri_nx, cl_nx, sq_nx = _networkx(s, o, n)
    assert np.array_equal(got["degree"], deg_nx) and np.array_equal(tri, tri_nx)
    assert np.array_equal(cl.view(np.int64), cl_nx.view(np.int64))
    assert np.array_equal(sq.view(np.int64), sq_nx.view(np.int64))


def test_host_array_input():
    s, o, n = GRAPHS["random_b"]
    from ampligraph_b200.engine import graph_counts
    got = graph_counts(np.stack([s, s, o], 1), n)  # a host array, on the current device
    _assert_equal({k: v.cpu().numpy() for k, v in got.items()}, graph_oracle.counts(s, o, n))


def _cfg2_graph():
    sys.path.insert(0, ROOT)
    import bench
    t = bench.synthetic_kg(14505, 237, 272115)
    return t[:, 0].astype(np.int64), t[:, 2].astype(np.int64), 14505


def test_cfg2_graph_and_determinism():
    s, o, n = _cfg2_graph()
    got = _gpu(s, o, n)
    _assert_equal(got, graph_oracle.counts(s, o, n))
    again = _gpu(s, o, n)
    _assert_equal(again, got)


def test_workspace_path_above_shared_bound():
    """More nodes than fit in shared memory: each CTA counts in its own slice of the workspace."""
    n = _shared_bound() + 5000
    rng = np.random.default_rng(11)
    m = 4 * n
    w = 1.0 / np.arange(1, n + 1) ** 0.7
    p = w / w.sum()
    s, o = rng.choice(n, m, p=p), rng.choice(n, m, p=p)
    s[:100] = o[:100]
    from ampligraph_b200 import _lib
    assert _lib.load().kge_graph_workspace_bytes(n) > 256 + 4 * n  # the workspace path is taken
    got = _gpu(s, o, n)
    _assert_equal(got, graph_oracle.counts(s, o, n))
    _assert_equal(_gpu(s, o, n), got)


@pytest.mark.parametrize("m", [300, 70000])
def test_complete_bipartite_needs_int64(m):
    """K_{2,m}: at m = 70,000 a hub's sq = C(m, 2) > 2^31, and the graph is above the shared-memory bound."""
    s, o, want = graph_oracle.complete_bipartite_2(m)
    got = _gpu(s, o, m + 2)
    _assert_equal(got, want)
    if m == 70000:
        assert got["sq"][0] > 2 ** 31


def test_invalid_arguments():
    from ampligraph_b200 import _lib
    from ampligraph_b200.engine import graph_counts
    lib = _lib.load()
    assert lib.kge_graph_workspace_bytes(-1) == 0
    with pytest.raises(ValueError, match="workspace"):
        z = torch.zeros(8, dtype=torch.int64, device="cuda")
        _lib.check(lib.kge_graph_counts(z.data_ptr(), z.data_ptr(), z.data_ptr(), 3, z.data_ptr(), z.data_ptr(),
                                        z.data_ptr(), None, 0, None))
    with pytest.raises(ValueError, match="node ids"):
        graph_counts(np.array([[0, 0, 5]]), 3)


@pytest.mark.parametrize("case", [c for c in GOLDEN["candidates"] if c["strategy"] in CLUSTER], ids=_case_id)
def test_cluster_strategies_match_reference(case):
    check_case(case)


# -- discover_facts ---------------------------------------------------------------------------------------------------

def _fitted(X, seed=0, epochs=20):
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    model = ScoringBasedEmbeddingModel(eta=5, k=10, scoring_type="ComplEx", seed=seed)
    model.compile(optimizer="adam", loss="multiclass_nll")
    model.fit(X, batch_size=64, epochs=epochs, verbose=False)
    return model


def _restated(X, model, rel_list, top_n, strategy, max_candidates, seed):
    """The reference's loop (discovery.py:241-271) on the reference's candidates: one evaluate per relation."""
    from ampligraph_b200 import discovery
    cands, ranks = [], []
    for rel in rel_list:
        c = discovery.generate_candidates(X, strategy, rel, max_candidates, seed=seed)
        if len(c) == 0:
            continue
        r = np.mean(model.evaluate(c, use_filter={"test": X}, corrupt_side="s,o", verbose=False), axis=1)
        cands.append(c[r <= top_n])
        ranks.append(r[r <= top_n])
    return cands, ranks


def test_discover_facts_reference_errors():
    """The reference's test_discover_facts."""
    from ampligraph_b200.discovery import discover_facts
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    X = np.array([['a', 'y', 'b'], ['b', 'y', 'a'], ['a', 'y', 'c'], ['c', 'y', 'a'], ['a', 'y', 'd'],
                  ['c', 'y', 'd'], ['b', 'y', 'c'], ['f', 'y', 'e']])
    model = ScoringBasedEmbeddingModel(eta=5, k=10, scoring_type='ComplEx')
    model.compile(optimizer='adam', loss='multiclass_nll')
    with pytest.raises(ValueError):
        discover_facts(X, model)
    model.fit(X, epochs=10, batch_size=3, verbose=False)
    with pytest.raises(ValueError):
        discover_facts(X, model, strategy='error')
    with pytest.raises(ValueError):
        discover_facts(X, model, strategy='random_uniform', target_rel='error')


@pytest.mark.parametrize("strategy", ["random_uniform", "graph_degree", "cluster_squares"])
def test_discover_facts_equals_reference_loop(strategy):
    from ampligraph_b200.discovery import discover_facts
    X = DATASETS["zipf"]
    model = _fitted(X)
    got, ranks = discover_facts(X, model, top_n=100, strategy=strategy, max_candidates=80, target_rel="r2", seed=3)
    cands, want = _restated(X, model, [["r2"]], 100, strategy, 80, 3)
    assert got.dtype == object and ranks.dtype == np.float64
    assert np.array_equal(got, cands[0]) and np.array_equal(ranks, want[0])
    assert len(got) > 0


def test_discover_facts_all_relations_stacked():
    """target_rel=None: every relation in the indexer's order, stacked with vstack even when the counts differ."""
    from ampligraph_b200.discovery import discover_facts
    X = DATASETS["zipf"]
    model = _fitted(X)
    rels = list(model.data_indexer.rel_labels)
    got, ranks = discover_facts(X, model, top_n=40, strategy="entity_frequency", max_candidates=60, seed=1)
    cands, want = _restated(X, model, rels, 40, "entity_frequency", 60, 1)
    assert len({len(c) for c in cands}) > 1  # the reference's np.hstack would raise here
    assert np.array_equal(got, np.vstack(cands)) and np.array_equal(ranks, np.concatenate(want))


def _with_unseen(X):
    """X plus 40 triples whose subject and object are entities a model fitted on X has never seen."""
    new = np.array([["new_s%d" % i, "r1", "new_o%d" % i] for i in range(40)])
    return np.concatenate([X, new])


def test_discover_facts_drops_unseen_entities(caplog):
    from ampligraph_b200.discovery import discover_facts, generate_candidates
    X = DATASETS["zipf"]
    model = _fitted(X)
    X2 = _with_unseen(X)
    with caplog.at_level(logging.WARNING, logger="ampligraph_b200.discovery"):
        got, ranks = discover_facts(X2, model, top_n=10 ** 6, strategy="random_uniform", max_candidates=400,
                                    target_rel="r1", seed=2)
    assert "not seen by the model" in caplog.text
    seen = set(model.data_indexer.ent_labels.tolist())
    cands = generate_candidates(X2, "random_uniform", ["r1"], 400, seed=2)
    keep = np.array([r[0] in seen and r[2] in seen for r in cands])
    assert not keep.all() and np.array_equal(got, cands[keep]) and len(ranks) == keep.sum()


def test_discover_facts_float_max_candidates():
    from ampligraph_b200.discovery import discover_facts
    X = DATASETS["zipf"]
    model = _fitted(X)
    got, ranks = discover_facts(X, model, top_n=10 ** 6, max_candidates=0.02, target_rel="r0", seed=5)
    want = discover_facts(X, model, top_n=10 ** 6, max_candidates=int(0.02 * len(X)), target_rel="r0", seed=5)
    assert len(got) == int(0.02 * len(X))
    assert np.array_equal(got, want[0]) and np.array_equal(ranks, want[1])
