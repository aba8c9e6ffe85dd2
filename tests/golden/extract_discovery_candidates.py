#!/usr/bin/env python
"""Run the reference's generate_candidates and _setdiff2d and record their outputs as JSON.

The reference's ampligraph/discovery/discovery.py imports only numpy, scipy, sklearn and networkx, so it is loaded by
path with importlib (no TensorFlow, no package import) and called as is.  Run it against a checkout of the reference;
the JSON it writes is committed, so the tests never need the reference itself.

    python tests/golden/extract_discovery_candidates.py <path to the reference checkout>

Output: tests/golden/discovery_candidates.json
  datasets:  name -> X as a list of [s, p, o] string rows
  candidates: one entry per call: dataset, strategy, target_rel, max_candidates, consolidate_sides, seed, and either
              "out" (the rows) or "error" (exception type name and message)
  setdiff2d:  A, B and the reference's _setdiff2d(A, B)
"""
import importlib.util
import json
import logging
import os
import sys

import numpy as np

if len(sys.argv) != 2:
    sys.exit(__doc__)
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "discovery_candidates.json")
spec = importlib.util.spec_from_file_location("reference_discovery",
                                              os.path.join(sys.argv[1], "ampligraph", "discovery", "discovery.py"))
ref = importlib.util.module_from_spec(spec)
spec.loader.exec_module(ref)
logging.disable(logging.WARNING)

STRATEGIES = ["random_uniform", "entity_frequency", "graph_degree", "cluster_coefficient", "cluster_triangles",
              "cluster_squares"]


def reference_test_x():
    """The 50-row X of the reference's test_generate_candidates."""
    return np.stack([["entity_{}".format(np.mod(x, 15)) for x in range(50)],
                     ["rel_{}".format(np.mod(x, 5)) for x in range(50)],
                     ["entity_{}".format(np.mod(x, 20)) for x in range(50)]], axis=1)


def zipf_kg(n_ent=300, n_rel=7, n=2000, seed=5):
    """Seeded Zipf(1) KG with 40 self-loops and 60 repeated triples."""
    rng = np.random.default_rng(seed)
    w = 1.0 / np.arange(1, n_ent + 1)
    cdf = np.cumsum(w / w.sum())
    perm = rng.permutation(n_ent)
    s = perm[np.searchsorted(cdf, rng.random(n - 60))]
    o = perm[np.searchsorted(cdf, rng.random(n - 60))]
    p = rng.integers(0, n_rel, n - 60)
    o[:40] = s[:40]
    X = np.stack([np.char.add("e", s.astype(str)), np.char.add("r", p.astype(str)), np.char.add("e", o.astype(str))], 1)
    return np.concatenate([X, X[rng.integers(0, len(X), 60)]])


def call(X, **kw):
    try:
        out = ref.generate_candidates(X, **kw)
        return {"out": [[str(v) for v in row] for row in out]}
    except Exception as e:  # recorded: the port must raise the same
        return {"error": [type(e).__name__, str(e)]}


def main():
    datasets = {"reference_test": reference_test_x(), "zipf": zipf_kg()}
    cases = []
    for name, X in datasets.items():
        rel = X[0, 1]
        for strategy in STRATEGIES:
            for consolidate_sides in (False, True):
                for seed in (0, 1916):
                    for max_candidates in (30, 0.3 if name == "reference_test" else 0.05):
                        kw = dict(strategy=strategy, target_rel=rel, max_candidates=max_candidates,
                                  consolidate_sides=consolidate_sides, seed=seed)
                        cases.append(dict(dataset=name, **kw, **call(X, **kw)))
        kw = dict(strategy="graph_degree", target_rel=[X[1, 1]], max_candidates=40, consolidate_sides=False, seed=3)
        cases.append(dict(dataset=name, **kw, **call(X, **kw)))
        kw = dict(strategy="random_uniform", target_rel="not_a_relation", max_candidates=20, consolidate_sides=False,
                  seed=3)
        cases.append(dict(dataset=name, **kw, **call(X, **kw)))
    rng = np.random.default_rng(9)
    setdiff = [{"A": [["a", "y", "b"], ["a", "y", "b"], ["c", "y", "d"]], "B": [["a", "y", "b"]]}]
    for _ in range(20):
        A = rng.integers(0, 3, (int(rng.integers(1, 14)), 3)).astype(str)
        B = rng.integers(0, 3, (int(rng.integers(1, 14)), 3)).astype(str)
        setdiff.append({"A": A.tolist(), "B": B.tolist()})
    for c in setdiff:
        c["out"] = ref._setdiff2d(np.array(c["A"]), np.array(c["B"])).tolist()
    with open(OUT, "w") as f:
        json.dump({"datasets": {k: v.tolist() for k, v in datasets.items()}, "candidates": cases,
                   "setdiff2d": setdiff}, f, separators=(",", ":"))
    print("%s: %d candidate cases, %d setdiff cases, %d bytes" % (OUT, len(cases), len(setdiff), os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
