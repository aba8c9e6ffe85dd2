"""CPU tests of the evaluation protocol (ampligraph_b200.evaluation): train_test_split_no_unseen and the combination
sequences of select_best_model_ranking against the reference's outputs in tests/golden/protocol.json
(tests/golden/extract_protocol.py), and filter_unseen_entities."""
import importlib.util
import json
import os
from types import SimpleNamespace

import numpy as np
import pytest

from ampligraph_b200 import evaluation as ev
from ampligraph_b200.datasets import DataIndexer

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
with open(os.path.join(GOLDEN, "protocol.json")) as f:
    FIX = json.load(f)
_spec = importlib.util.spec_from_file_location("extract_protocol", os.path.join(GOLDEN, "extract_protocol.py"))
extract = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(extract)  # for decode_grid, typed and digest; main() only runs as a script


def _dataset(name):
    X = FIX["datasets"][name]
    return np.array(X) if not name.endswith("_int") else np.array(X, dtype=np.int64)


@pytest.mark.parametrize("case", FIX["split"], ids=lambda c: "%s-%s-%s-%s" % (c["dataset"], c["test_size"], c["seed"],
                                                                              c["allow_duplication"]))
def test_split_matches_reference(case):
    X = _dataset(case["dataset"])
    state = np.random.get_state()
    kw = dict(test_size=case["test_size"], seed=case["seed"], allow_duplication=case["allow_duplication"],
              filtered_test_predicates=case["filtered_test_predicates"])
    if "error" in case:
        with pytest.raises(Exception) as e:
            ev.train_test_split_no_unseen(X, **kw)
        assert [type(e.value).__name__, str(e.value)] == case["error"]
    else:
        tr, te = ev.train_test_split_no_unseen(X, **kw)
        assert extract.digest(tr) == case["out"]["train"] and extract.digest(te) == case["out"]["test"]
        assert tr.dtype == X.dtype and te.dtype == X.dtype
        if "rows" in case["out"]:
            assert [tr.tolist(), te.tolist()] == case["out"]["rows"]
    rest = np.random.get_state()
    assert all(np.array_equal(a, b) for a, b in zip(state, rest))  # the global generator is untouched


def test_split_never_leaves_unseen():
    """The test set's entities and relations all occur in the train set, and no triple is lost."""
    X = _dataset("zipf")
    tr, te = ev.train_test_split_no_unseen(X, test_size=600, seed=9)
    assert len(tr) + len(te) == len(X)
    assert set(te[:, [0, 2]].ravel()) <= set(tr[:, [0, 2]].ravel()) and set(te[:, 1]) <= set(tr[:, 1])


@pytest.mark.parametrize("g", FIX["grids"], ids=lambda g: "%s-%s-%s" % (g["model_class"], g["max_combinations"],
                                                                        g["param_grid_random_seed"]))
def test_combinations_match_reference(g):
    grid = extract.decode_grid(g["grid"])
    before = _snapshot(grid)
    state = np.random.get_state()
    combos, n = ev._combinations(g["model_class"], grid, g["max_combinations"], g["param_grid_random_seed"])
    got = [extract.typed(c) for c in combos]
    assert n == g["n"]
    if g["ordered"]:
        assert got == g["combos"]
    else:  # the reference orders the product of two nested dicts by Python's string hashing
        key = lambda c: json.dumps(c, sort_keys=True)
        assert sorted(map(key, got)) == sorted(map(key, g["combos"]))
    assert _snapshot(grid) == before  # the caller's grid is untouched
    rest = np.random.get_state()
    assert all(np.array_equal(a, b) for a, b in zip(state, rest))


def _snapshot(grid):
    """A copy of a grid's structure holding the same leaf objects (callables compare by identity)."""
    return {k: _snapshot(v) if isinstance(v, dict) else v for k, v in grid.items()}


def test_random_combinations_interleaved_with_global_draws():
    """The user's draws from np.random between two combinations change neither the combinations nor the draws."""
    g = next(g for g in FIX["grids"] if g["model_class"] == "ComplEx" and g["max_combinations"] == 6)
    combos, _ = ev._combinations(g["model_class"], extract.decode_grid(g["grid"]), 6, 0)
    np.random.seed(123)
    want = np.random.uniform(size=6)
    np.random.seed(123)
    got, draws = [], []
    for c in combos:
        got.append(extract.typed(c))
        draws.append(np.random.uniform())
    assert got == g["combos"] and np.array_equal(draws, want)


def _fitted(labels=True):
    X = np.array([["a", "r", "b"], ["b", "r", "c"], ["c", "s", "a"]])
    if labels:
        return X, SimpleNamespace(data_indexer=DataIndexer(X), max_ent_size=3)
    return X, SimpleNamespace(data_indexer=False, max_ent_size=3)


def test_filter_unseen_entities_labels():
    _, model = _fitted()
    X = np.array([["a", "r", "c"], ["a", "r", "z"], ["z", "s", "b"], ["b", "q", "a"]])
    out = ev.filter_unseen_entities(X, model)
    assert out.tolist() == [["a", "r", "c"], ["b", "q", "a"]]  # relations are not checked, as in the reference
    assert out.dtype == object  # the reference returns a DataFrame's values
    kept = X[:1]
    assert ev.filter_unseen_entities(kept, model) is kept  # nothing removed: X itself


def test_filter_unseen_entities_ids():
    _, model = _fitted(labels=False)
    X = np.array([[0, 0, 2], [0, 1, 3], [5, 0, 1], [2, 0, 1]])
    assert ev.filter_unseen_entities(X, model).tolist() == [[0, 0, 2], [2, 0, 1]]
    kept = X[:1]
    assert ev.filter_unseen_entities(kept, model) is kept
    with pytest.raises(RuntimeError):
        ev.filter_unseen_entities(X, SimpleNamespace(data_indexer=True, max_ent_size=None))


def test_split_error_and_int_sizes():
    """Sizes the reference compares with == (a float is taken as a fraction only when it is a float)."""
    X = _dataset("doc")
    assert len(ev.train_test_split_no_unseen(X, test_size=np.int64(2))[1]) == 2
    with pytest.raises(Exception, match="Cannot create a test split"):
        ev.train_test_split_no_unseen(X, test_size=100)


def test_eta_as_int32():
    assert ev._as_int32(np.int64(3)) == 3 and isinstance(ev._as_int32(np.int64(3)), np.int32)
    assert ev._as_int32(3) == 3  # the reference's .astype(np.int32) fails on a Python int; accepted here
    with pytest.raises(TypeError):
        ev._as_int32("3")
