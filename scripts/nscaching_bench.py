#!/usr/bin/env python
"""NSCaching benchmark (development aid; DESIGN.md 3.20, 5): kge_nscaching_step (csrc/kge_nscaching.cu) at two shapes of
bench.py's workloads on one GPU, on their seeded synthetic KGs:
  cfg2  ComplEx k = 200, eta = 10, B = 27,212 (14,505 entities, 272,115 triples)
  cfg4  RotatE k = 200, eta = 30, B = 10,791, cfg4's table (123,182 entities, 1,079,040 triples), unsharded

- The NSCaching call alone (refresh + draw, caches warmed by earlier calls) at N1 = N2 = 50 and at N1 = 200, N2 = 312:
  its device time (CUDA events around each call, median), the refreshed rows, and the achieved rate of the row bytes it
  gathers: per refreshed row (count + N2) candidate rows and the query's s, p and o rows, ld floats each.
- The full deferred training step (forward_backward(defer=True) + apply_gradients) with 'nscaching' (N1 = N2 = 50),
  'uniform' (in-kernel draws) and 'bernoulli', alternated in one run.
Prints the GPU and its power limit first: every number depends on both.

    python scripts/nscaching_bench.py [--iters N] [--rounds R] [--out FILE.json]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import measure  # noqa: E402

SETTINGS = [(50, 50), (200, 312)]


def shape(cfg_name, a, res):
    import bench
    from ampligraph_b200.datasets import negative_sampler_tables, nscaching_tables
    from ampligraph_b200.engine import KGEEngine, NegativeSamplerTables, NSCache
    c = bench.WORKLOADS[cfg_name]
    E, R, B, eta = c["n_ent"], c["n_rel"], c["batch"], c["eta"]
    kg = bench.synthetic_kg(E, R, c["n_triples"])
    eng = KGEEngine(c["model"], c["k"], eta, E, R, loss=c["loss"], loss_params=c["loss_params"], optimizer="adam",
                    optimizer_params={"learning_rate": c["lr"]})
    eng.init_glorot_uniform(seed=1)
    eng.set_hot_entities(triples=kg)
    data = torch.as_tensor(kg).cuda().contiguous()
    batch = data[:B]
    host = nscaching_tables(kg, E, R, B)
    ld = eng.lib.kge_internal_k(eng.h)  # dense width; the padded row is the same for k = 200
    out = {"workload": "%s: %s k=%d, eta=%d, B=%d, %d entities" % (cfg_name, c["model"], c["k"], eta, B, E),
           "alone": {}, "step_ms": {}}
    for n1, n2 in SETTINGS:
        cache = NSCache(host, n1, n2, eng.device)
        key_rows, update = cache.batch(0, B)
        state = {"step": 0}

        def call():
            eng.nscaching_negatives(batch, key_rows, update, cache, 0, state["step"])
            state["step"] += 1
        for _ in range(3):  # fill the caches: the timed calls refresh full rows
            call()
        ms = measure.per_call_ms(call, a.iters, 2)
        flagged = update.bool()
        rows = int(flagged.sum())
        cached = sum(int(cache.count[side][key_rows[:, side][flagged[:, side]].long()].sum()) for side in (0, 1))
        mean_count = cached / max(rows, 1)  # the refreshed rows' cached ids, as the next call finds them
        gathered = rows * (mean_count + n2 + 3) * ld * 4
        med = float(np.median(ms))
        out["alone"]["N1=%d,N2=%d" % (n1, n2)] = {
            "median_ms": med, "p10_ms": float(np.percentile(ms, 10)), "p90_ms": float(np.percentile(ms, 90)),
            "refreshed_rows": rows, "mean_cached_per_refreshed_row": mean_count, "gathered_GB": gathered / 1e9,
            "gathered_GB_per_s": gathered / 1e9 / (med / 1e3)}
        eng.read_negative_misses()
        print(json.dumps({cfg_name: out["alone"]}), flush=True)

    cache = NSCache(host, 50, 50, eng.device)
    key_rows, update = cache.batch(0, B)
    bern = NegativeSamplerTables(negative_sampler_tables(kg, E, R, "bernoulli"), 1, eng.device)
    state = {"step": 0}

    def step(kind):
        s = state["step"]
        if kind == "uniform":
            negs = None
        elif kind == "bernoulli":
            negs = eng.sample_negatives(batch, bern, 0, s)
        else:
            negs = eng.nscaching_negatives(batch, key_rows, update, cache, 0, s)
        eng.forward_backward(batch, negs, seed=0, step=s, defer=True)
        eng.apply_gradients()
        state["step"] += 1
    kinds = ["uniform", "bernoulli", "nscaching"]
    times = measure.alternated({k: lambda k=k: step(k) for k in kinds}, a.rounds, a.iters, 2)
    for k in kinds:
        out["step_ms"][k] = {"median": float(np.median(times[k])), "p10": float(np.percentile(times[k], 10)),
                             "p90": float(np.percentile(times[k], 90))}
    print(json.dumps({cfg_name: out["step_ms"]}), flush=True)
    eng.read_negative_misses()
    eng.close()
    res[cfg_name] = out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("nscaching_bench.py needs a CUDA device: there is no CPU measurement")
    res = {"gpu": measure.card()}
    print(res["gpu"], flush=True)
    for cfg_name in ("cfg2", "cfg4"):
        shape(cfg_name, a, res)
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
