"""Time the evaluation protocol (ampligraph_b200.evaluation).

  split       train_test_split_no_unseen on FB15K-237-shaped Zipf graphs of 272 k and 1.08 M triples (14,505 entities,
              237 relations), test_size 20,466; with --reference, the reference's own per-triple loop on the same
              inputs (loaded as tests/golden/extract_protocol.py loads it).  Host only.
  validation  one validation inside fit at cfg2's size (ComplEx k=200, eta 10, string labels; 272 k train, 17.5 k valid,
              20.5 k test; X_valid[::2] ranked on both sides with the {train, valid, test} filter): as every validation
              did before fit built the filter once (index the three datasets and build a FilterIndex, then rank), and
              with the FilterIndex fit now builds before its epoch loop.  Wall time, GPU synchronised.
  search      one small select_best_model_ranking end to end (4 candidates, early stopping), wall time.

  python scripts/protocol_bench.py [--reference PATH] [--host-only] [--reps 5]
Prints the card and its power limit, then one JSON line per measurement."""
import argparse
import importlib.util
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from ampligraph_b200.evaluation import train_test_split_no_unseen  # noqa: E402

E, R = 14505, 237


def zipf_labels(n, seed):
    rng = np.random.default_rng(seed)
    w = 1.0 / np.arange(1, E + 1)
    cdf = np.cumsum(w / w.sum())
    perm = rng.permutation(E)
    s, o = perm[np.searchsorted(cdf, rng.random(n))], perm[np.searchsorted(cdf, rng.random(n))]
    p = rng.integers(0, R, n)
    return np.stack([np.char.add("e", s.astype(str)), np.char.add("r", p.astype(str)), np.char.add("e", o.astype(str))], 1)


def wall(fn, reps, sync=None):
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        if sync is not None:
            sync()
        times.append(time.perf_counter() - t0)
    return float(np.median(times)) * 1e3, float(np.min(times)) * 1e3


def bench_split(args):
    ref = None
    if args.reference:
        spec = importlib.util.spec_from_file_location("extract_protocol",
                                                      os.path.join(ROOT, "tests", "golden", "extract_protocol.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        ref = mod.load_reference(args.reference)
    for n in (272115, 1088460):
        X = zipf_labels(n, 0)
        med, best = wall(lambda: train_test_split_no_unseen(X, test_size=20466, seed=0), args.reps)
        out = {"what": "split", "triples": n, "test_size": 20466, "ms_median": round(med, 1), "ms_min": round(best, 1)}
        if ref is not None:
            out["reference_ms"] = round(wall(lambda: ref.train_test_split_no_unseen(X, test_size=20466, seed=0), 1)[0], 1)
            a, b = train_test_split_no_unseen(X, test_size=20466, seed=0), ref.train_test_split_no_unseen(X, 20466, 0)
            out["equal"] = bool(all(np.array_equal(x, y) for x, y in zip(a, b)))
        print(json.dumps(out), flush=True)


def bench_gpu(args):
    import measure
    import torch
    from ampligraph_b200.evaluation import select_best_model_ranking
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    print(measure.card())
    X = zipf_labels(272115 + 17535 + 20466, 1)
    train, valid, test = X[:272115], X[272115:272115 + 17535], X[272115 + 17535:]
    m = ScoringBasedEmbeddingModel(eta=10, k=200, scoring_type="ComplEx", seed=0)
    m.compile(optimizer="adam", loss="self_adversarial")
    m.fit(train, batch_size=27212, epochs=1, verbose=False)
    filt = {"train": train, "valid": valid, "test": test}
    v = valid[::2]
    sync = torch.cuda.synchronize

    def before():  # what each validation did: index the filter datasets, build the FilterIndex, rank
        m.evaluate(v, batch_size=10, verbose=False, use_filter=filt)
    t0 = time.perf_counter()
    kept = m._build_filter(filt, None)  # once per fit, before the epoch loop
    build_ms = (time.perf_counter() - t0) * 1e3

    def after():
        m.evaluate(v, batch_size=10, verbose=False, use_filter=filt, _filter_index=kept)
    before()
    after()
    sync()
    b_med, b_min = wall(before, args.reps, sync)
    a_med, a_min = wall(after, args.reps, sync)
    print(json.dumps({"what": "validation", "queries": len(v), "sides": 2, "before_ms_median": round(b_med, 1),
                      "before_ms_min": round(b_min, 1), "after_ms_median": round(a_med, 1),
                      "after_ms_min": round(a_min, 1), "filter_build_once_ms": round(build_ms, 1)}), flush=True)
    del m
    Xs = zipf_labels(30000, 2)
    Xs[:, 0] = np.char.add("e", (np.char.lstrip(Xs[:, 0], "e").astype(int) % 2000).astype(str))
    Xs[:, 2] = np.char.add("e", (np.char.lstrip(Xs[:, 2], "e").astype(int) % 2000).astype(str))
    rest, te = train_test_split_no_unseen(Xs, test_size=1000, seed=0)
    tr, va = train_test_split_no_unseen(rest, test_size=1000, seed=1)
    grid = {"batch_size": [2800], "epochs": [50], "k": [50, 100], "eta": [5, 10], "loss": ["multiclass_nll"],
            "optimizer_params": {"learning_rate": [0.005]}}
    t0 = time.perf_counter()
    out = select_best_model_ranking("ComplEx", tr, va, te, grid,
                                    early_stopping_params={"check_interval": 5, "stop_interval": 2})
    sync()
    secs = time.perf_counter() - t0
    print(json.dumps({"what": "search", "train": len(tr), "candidates": len(out[5]), "seconds": round(secs, 2),
                      "best_epochs": out[1]["early_stopping_epoch"],
                      "selection_mrr": [round(h["results"].get("mrr", float("nan")), 4) for h in out[5]],
                      "test_mrr": round(out[4]["mrr"], 4)}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default=None, help="a checkout of the reference, to time its split loop")
    ap.add_argument("--host-only", action="store_true")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    bench_split(args)
    if not args.host_only:
        bench_gpu(args)


if __name__ == "__main__":
    main()
