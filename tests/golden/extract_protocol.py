#!/usr/bin/env python
"""Run the reference's train_test_split_no_unseen and its hyper-parameter combination generators and record their
outputs as JSON.

The reference's ampligraph/evaluation/protocol.py imports TensorFlow (only to build a Keras EarlyStopping inside
select_best_model_ranking) and its metrics from the package.  It is loaded by path with importlib, under a stub
`tensorflow` module and a stub `ampligraph.evaluation` package whose metrics come from the reference's metrics.py (which
needs only numpy); the functions recorded here never touch the stubs.  The JSON it writes is committed, so the tests
never need the reference itself.

    python tests/golden/extract_protocol.py <path to the reference checkout>

Output: tests/golden/protocol.json
  datasets: name -> X as a list of rows (strings, or ints for the *_int datasets)
  split:    one entry per call: dataset, test_size, seed, allow_duplication, filtered_test_predicates, and either
            "out" ({"train": [n, sha256], "test": [n, sha256]}, with the rows themselves for the small datasets) or
            "error" (exception type name and message)
  grids:    one entry per grid: model_class, the grid (callables as ["@uniform" | "@randint", a, b], see decode_grid),
            max_combinations, param_grid_random_seed, "ordered" (False when the reference's order depends on Python's
            string hashing: a grid search over two nested dicts), n (how many combinations select_best_model_ranking
            walks) and "combos", each a dict whose leaves are [type name, value]
"""
import hashlib
import importlib.util
import json
import os
import sys
import types
from itertools import islice

import numpy as np

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "protocol.json")
SMALL = 40  # datasets of at most this many rows keep their output rows in the JSON


def load_reference(root):
    """The reference's evaluation/protocol.py as a module, with stub tensorflow and ampligraph.evaluation modules."""
    sys.modules.setdefault("tensorflow", types.ModuleType("tensorflow"))
    if "tqdm" not in sys.modules:
        try:
            import tqdm  # noqa: F401
        except ImportError:
            stub = types.ModuleType("tqdm")
            stub.tqdm = lambda it, **kw: it
            sys.modules["tqdm"] = stub
    pkg = types.ModuleType("ampligraph")
    pkg.__path__ = []
    ev = types.ModuleType("ampligraph.evaluation")
    ev.__path__ = []
    sys.modules["ampligraph"], sys.modules["ampligraph.evaluation"] = pkg, ev
    mods = {}
    for name in ("metrics", "protocol"):
        spec = importlib.util.spec_from_file_location("ampligraph.evaluation." + name,
                                                      os.path.join(root, "ampligraph", "evaluation", name + ".py"))
        mods[name] = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mods[name])
        if name == "metrics":
            for f in ("hits_at_n_score", "mr_score", "mrr_score"):
                setattr(ev, f, getattr(mods[name], f))
    return mods["protocol"]


def decode_grid(spec):
    """JSON grid -> param_grid: ["@uniform", a, b] and ["@randint", a, b] become callables drawing from np.random."""
    if isinstance(spec, dict):
        return {k: decode_grid(v) for k, v in spec.items()}
    if isinstance(spec, list) and spec and spec[0] == "@uniform":
        return lambda: np.random.uniform(spec[1], spec[2])
    if isinstance(spec, list) and spec and spec[0] == "@randint":
        return lambda: np.random.randint(spec[1], spec[2])
    return spec


def typed(v):
    """A combination with every leaf as [type name, value]."""
    if isinstance(v, dict):
        return {k: typed(x) for k, x in v.items()}
    return [type(v).__name__, v.item() if isinstance(v, np.generic) else v]


def digest(A):
    """[rows, sha256 of the rows as tab-separated text] of a split output."""
    text = "\n".join("\t".join(str(x) for x in row) for row in np.asarray(A).tolist())
    return [len(A), hashlib.sha256(text.encode()).hexdigest()]


def docstring_x():
    return np.array([["a", "y", "b"], ["f", "y", "e"], ["b", "y", "a"], ["a", "y", "c"], ["c", "y", "a"],
                     ["a", "y", "d"], ["c", "y", "d"], ["b", "y", "c"], ["f", "y", "e"]])


def zipf_kg(n_ent=300, n_rel=7, n=2000, seed=5, labels=True):
    """Seeded Zipf(1) KG with 40 self-loops and 60 repeated triples."""
    rng = np.random.default_rng(seed)
    w = 1.0 / np.arange(1, n_ent + 1)
    cdf = np.cumsum(w / w.sum())
    perm = rng.permutation(n_ent)
    s = perm[np.searchsorted(cdf, rng.random(n - 60))]
    o = perm[np.searchsorted(cdf, rng.random(n - 60))]
    p = rng.integers(0, n_rel, n - 60)
    o[:40] = s[:40]
    X = np.stack([s, p, o], 1)
    X = np.concatenate([X, X[rng.integers(0, len(X), 60)]])
    if not labels:
        return X
    return np.stack([np.char.add("e", X[:, 0].astype(str)), np.char.add("r", X[:, 1].astype(str)),
                     np.char.add("e", X[:, 2].astype(str))], 1)


def small_kgs(count=12, seed=11):
    """Tiny random graphs: few entities, so self-loops, repeats and failing sizes are common."""
    rng = np.random.default_rng(seed)
    out = {}
    for i in range(count):
        ne, nr, n = int(rng.integers(2, 20)), int(rng.integers(1, 4)), int(rng.integers(5, 40))
        out["small%d" % i] = np.stack([rng.integers(0, ne, n), rng.integers(0, nr, n), rng.integers(0, ne, n)], 1).astype(str)
    return out


GRIDS = [
    dict(model_class="ComplEx", max_combinations=None, param_grid_random_seed=0,
         grid={"batch_size": [100], "k": [8, 16], "eta": [2, 3], "loss": ["pairwise", "nll"],
               "loss_params": {"margin": [1, 2]}, "seed": 0, "verbose": False}),
    dict(model_class="ComplEx", max_combinations=5, param_grid_random_seed=0,
         grid={"batch_size": [100], "k": [8, 16], "eta": [2, 3], "loss": ["pairwise", "nll"],
               "loss_params": {"margin": [1, 2]}, "seed": 0, "verbose": False}),
    dict(model_class="TransE", max_combinations=100, param_grid_random_seed=3,
         grid={"k": [8, 16], "eta": [2, 3], "optimizer": "adam", "optimizer_params": {"lr": [0.1, 0.01, 0.001]}}),
    dict(model_class="DistMult", max_combinations=None, param_grid_random_seed=0,
         grid={"k": [8, 8, 16], "eta": 2, "optimizer_params": {"lr": [0.1, 0.1]}, "regularizer": ["LP", None]}),
    dict(model_class="DistMult", max_combinations=4, param_grid_random_seed=1,
         grid={"k": [8, 8, 16], "eta": 2, "optimizer_params": {"lr": [0.1, 0.1]}, "regularizer": ["LP", None]}),
    dict(model_class="ComplEx", max_combinations=6, param_grid_random_seed=0,
         grid={"k": [8, 16, 32], "eta": ["@randint", 1, 10], "regularizer": ["LP", None],
               "regularizer_params": {"p": [1, 3], "lambda": ["@uniform", 1e-5, 1e-3]},
               "optimizer": ["adagrad", "adam"], "optimizer_params": {"lr": ["@uniform", 1e-4, 1e-2]}}),
    dict(model_class="HolE", max_combinations=20, param_grid_random_seed=7,
         grid={"batch_size": [50, 100], "epochs": [5], "k": [4, 8], "eta": [1, 2, 5],
               "loss": ["pairwise", "multiclass_nll"], "loss_params": {"margin": [0.5, 1.0]},
               "optimizer_params": {"lr": [0.01, 0.001]}}),
    dict(model_class="HolE", max_combinations=None, param_grid_random_seed=0,
         grid={"k": [4, 8], "eta": [1, 2], "loss_params": {"margin": [0.5, 1.0]},
               "optimizer_params": {"lr": [0.01, 0.001]}}),
]


def split_cases(datasets):
    cases = []
    add = lambda name, **kw: cases.append(dict(dataset=name, **{"test_size": 100, "seed": 0, "allow_duplication": False,
                                                                 "filtered_test_predicates": None, **kw}))
    for seed in (0, 1, 2):
        add("doc", test_size=2, seed=seed)
    add("doc", test_size=0.25)
    add("doc", test_size=6)
    add("doc", test_size=6, allow_duplication=True)
    add("doc", test_size=2, filtered_test_predicates=["y"])
    add("doc", test_size=0)
    add("doc", test_size=0, allow_duplication=True)
    for name in ("zipf", "zipf_int"):
        rels = sorted(set(datasets[name][:, 1].tolist()))
        for seed, ts in ((0, 100), (7, 500), (0, 0.1), (3, 0.3), (0, 1500)):
            add(name, test_size=ts, seed=seed)
        add(name, test_size=1500, seed=1, allow_duplication=True)
        add(name, test_size=50, seed=4, filtered_test_predicates=rels[:3])
        add(name, test_size=0.2, seed=5, filtered_test_predicates=rels[1:2])
        add(name, test_size=5000, seed=5, filtered_test_predicates=rels[1:2], allow_duplication=True)
    add("zipf", test_size=10, filtered_test_predicates=["not_a_relation"])
    add("zipf", test_size=0.001, allow_duplication=True)
    rng = np.random.default_rng(2)
    for name in datasets:
        if name.startswith("small"):
            n = len(datasets[name])
            add(name, test_size=int(rng.integers(1, n)), seed=int(rng.integers(0, 1000)),
                allow_duplication=bool(rng.integers(0, 2)))
    return cases


def main():
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    ref = load_reference(sys.argv[1])
    datasets = {"doc": docstring_x(), "zipf": zipf_kg(), "zipf_int": zipf_kg(labels=False), **small_kgs()}
    cases = split_cases(datasets)
    state = np.random.get_state()
    for c in cases:
        X = datasets[c["dataset"]]
        try:
            tr, te = ref.train_test_split_no_unseen(X, test_size=c["test_size"], seed=c["seed"],
                                                    allow_duplication=c["allow_duplication"],
                                                    filtered_test_predicates=c["filtered_test_predicates"])
            c["out"] = {"train": digest(tr), "test": digest(te)}
            if len(X) <= SMALL:
                c["out"]["rows"] = [tr.tolist(), te.tolist()]
        except Exception as e:  # recorded: the port must raise the same
            c["error"] = [type(e).__name__, str(e)]
    grids = []
    for g in GRIDS:
        grid = decode_grid(g["grid"])
        grid["model_name"] = g["model_class"]
        ref._scalars_into_lists(grid)
        total = 1
        for v in grid.values():
            if isinstance(v, list):
                total *= len(v)
            elif isinstance(v, dict):
                total *= int(np.prod([len(x) for x in v.values() if isinstance(x, list)]))
        if g["max_combinations"] is None:
            n, combos = total, list(ref._next_hyperparam(grid))
        else:
            n = int(np.min([total, g["max_combinations"]]))
            np.random.seed(g["param_grid_random_seed"])
            combos = list(islice(ref._next_hyperparam_random(grid), n))
        nested = sum(isinstance(v, dict) for v in g["grid"].values())
        grids.append(dict(g, n=n, ordered=g["max_combinations"] is not None or nested < 2,
                          combos=[typed(c) for c in combos]))
    np.random.set_state(state)
    with open(OUT, "w") as f:
        json.dump({"datasets": {k: v.tolist() for k, v in datasets.items()}, "split": cases, "grids": grids}, f,
                  separators=(",", ":"))
    print("%s: %d split cases (%d errors), %d grids, %d bytes" % (OUT, len(cases), sum("error" in c for c in cases),
                                                                len(grids), os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
