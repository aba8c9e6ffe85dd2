"""CPU tests (no GPU) of relation prediction (side 'p'): the (s, o) -> relations group of FilterIndex, the argument
errors of the facade and the C-ABI, and the relation-side oracle (tests/relation_oracle.py) against a numpy
restatement."""
import os

import numpy as np
import pytest

import relation_oracle


def _set_lookup(triples, queries, position_of=None):
    """Python-set restatement of FilterIndex.lookup(queries, 'p', position_of): per query, the sorted relations r with
    (s, r, o) in triples, mapped to candidate positions (those without one dropped)."""
    known = {}
    for s, r, o in {tuple(int(v) for v in t) for t in triples}:
        known.setdefault((s, o), set()).add(r)
    out = []
    for s, _, o in queries:
        rs = sorted(known.get((int(s), int(o)), ()))
        if position_of is not None:
            rs = [int(position_of[r]) for r in rs if position_of[r] >= 0]
        out.append(rs)
    return out


def test_filter_index_relation_lookup():
    from ampligraph_b200.datasets import FilterIndex
    rng = np.random.default_rng(5)
    E, R = 9, 6
    for n in (0, 1, 40, 300):
        triples = np.stack([rng.integers(0, E, n), rng.integers(0, R, n), rng.integers(0, E, n)], 1)
        triples = np.concatenate([triples, triples[: n // 3]])  # repeats count once
        fi = FilterIndex(triples, E)
        assert fi._rel is None  # built on the first 'p' lookup only
        queries = np.stack([rng.integers(0, E, 50), rng.integers(0, R, 50), rng.integers(0, E, 50)], 1)
        queries[:10] = triples[:10] if n >= 10 else queries[:10]
        sub = rng.choice(R, 4, replace=False)
        position_of = np.full(R, -1, np.int64)
        position_of[sub] = np.arange(4)
        for pos in (None, position_of):
            off, ids = fi.lookup(queries, "p", pos)
            want = _set_lookup(triples, queries, pos)
            assert off.dtype == np.int64 and ids.dtype == np.int32 and len(off) == len(queries) + 1
            assert [ids[off[i]:off[i + 1]].tolist() for i in range(len(queries))] == want
        # the entity sides are untouched by the relation group
        off_o, ids_o = fi.lookup(queries, "o")
        assert off_o[-1] == sum(len({t[2] for t in triples if t[0] == q[0] and t[1] == q[1]}) for q in queries)


def test_argument_errors():
    from ampligraph_b200.discovery import query_topn_batch
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    X = np.array([["a", "r", "b"], ["b", "q", "c"]], dtype=object)
    m = ScoringBasedEmbeddingModel(eta=1, k=4, scoring_type="TransE")
    with pytest.raises(ValueError, match="entities_subset"):
        m.evaluate(X, corrupt_side="p", entities_subset=["a"])
    for side in ("s", "o"):
        with pytest.raises(ValueError, match="rels_to_consider"):
            query_topn_batch(m, X, side=side, rels_to_consider=["r"])
    with pytest.raises(ValueError, match="ents_to_consider"):
        query_topn_batch(m, X, side="p", ents_to_consider=["a"])
    with pytest.raises(ValueError, match="'s', 'o' or 'p'"):
        query_topn_batch(m, X, side="x")


def test_sharded_rank_refuses_the_relation_side():
    """The relation table is replicated, never sharded: kge_rank_sharded refuses side P before it looks at anything
    else (so no handle or GPU is needed to see it)."""
    from ampligraph_b200 import _lib
    if not os.path.exists(_lib.SO_PATH):
        _lib.build()
    lib = _lib.load()
    assert _lib.SIDES["p"] == 2
    rc = lib.kge_rank_sharded(None, None, 0, _lib.SIDES["p"], 0, None, None, 4, None, None, 0, None, None, None, 0, None)
    assert rc == _lib.KGE_ERR_INVALID_ARGUMENT and b"relation" in lib.kge_last_error()
    with pytest.raises(ValueError, match="relation side"):
        _lib.check(rc)


def _transe_score(ent, rel, t):
    """TransE's canonical chain in numpy fp32, one rounding per operation: acc = acc + |(s + p) - o| over the columns."""
    s, p, o = ent[t[:, 0]], rel[t[:, 1]], ent[t[:, 2]]
    acc = np.zeros(len(t), np.float32)
    for d in range(ent.shape[1]):
        acc = (acc + np.abs((s[:, d] + p[:, d]) - o[:, d])).astype(np.float32)
    return -acc


def test_relation_oracle_vs_numpy():
    """The oracle's score grid is the canonical score of every completed (s, r, o); its counts follow the entity sides'
    rules (strategies, '<=' filter, window) -- checked against a numpy loop on TransE, whose chain numpy states exactly."""
    rng = np.random.default_rng(8)
    E, R, k, b = 30, 11, 7, 25
    ent = (rng.integers(-4, 5, (E, k)) / 8).astype(np.float32)  # coarse: quantised ties
    rel = (rng.integers(-4, 5, (R, k)) / 8).astype(np.float32)
    t = np.stack([rng.integers(0, E, b), rng.integers(0, R, b), rng.integers(0, E, b)], 1).astype(np.int32)
    cand = np.arange(R)
    full = np.stack([np.repeat(t[:, 0], R), np.tile(cand, b), np.repeat(t[:, 2], R)], 1)
    grid = _transe_score(ent, rel, full).reshape(b, R)
    got = relation_oracle.score_grid("TransE", ent, rel, t, cand)
    assert (got.view(np.uint32) == grid.view(np.uint32)).all()
    qpos = relation_oracle.quantise(_transe_score(ent, rel, t))
    qc = relation_oracle.quantise(grid)
    filters = [list(rng.integers(-2, R + 3, rng.integers(0, 6))) + [int(t[i, 1])] * (i % 3) for i in range(b)]
    windows = [(None, 0, None), (None, 3, 5), (np.array([7, 2, 9, 4]), 0, None)]
    ties = 0
    for cand_ids, begin, n_cand in windows:
        ids = relation_oracle.candidates(R, cand_ids, begin, n_cand)
        for strategy in ("worst", "best", "middle"):
            for filt in (None, filters):
                want = []
                for i in range(b):
                    c = qc[i, ids]
                    gt, eq = int((qpos[i] < c).sum()), int((qpos[i] == c).sum())
                    ties += eq
                    r = {"worst": gt + eq, "best": gt, "middle": gt + (eq + 1) // 2}[strategy]
                    for v in (filt[i] if filt is not None else []):
                        pos = v - (0 if cand_ids is not None else begin)
                        if 0 <= pos < len(ids):
                            r -= int(qpos[i] <= qc[i, ids[pos]])
                    want.append(r)
                got = relation_oracle.ranks("TransE", strategy, ent, rel, t, filt, cand_ids, begin, n_cand)
                assert got.tolist() == want, (strategy, begin, n_cand, cand_ids is not None, filt is not None)
    assert ties > 2 * b  # the coarse tables did force quantised ties
