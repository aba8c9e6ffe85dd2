#!/usr/bin/env python
"""Embedding-dropout benchmark (development aid): times kge_one_vs_all_step (sides s and o) and kge_k_vs_all_step
(side o) on the FB15k-237 shape -- 14,541 entities, 237 relations, ComplEx k = 200, B = 1,000 -- with embedding
dropout (p_ent, p_rel) = (0.4, 0.2) against (0, 0), alternating the two settings on one engine in one run, so that
both see the same clocks and neighbours.  Reported: the median step time of each setting (CUDA events around the call,
--rounds rounds of --iters steps each), the overhead, and the dropout kernels' own time (torch.profiler, a separate
pass).  Prints the GPU and its power limit first: every number depends on both.

    python scripts/dropout_bench.py [--iters N] [--rounds N] [--out FILE.json]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import measure  # noqa: E402

E, R, K_USER, B = 14541, 237, 200, 1000  # FB15k-237, ComplEx k = 200
DROPOUT = (0.4, 0.2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from ampligraph_b200.datasets import FilterIndex, k_vs_all_queries
    from ampligraph_b200.engine import KGEEngine

    info = measure.card()
    print(info)
    rng = np.random.default_rng(0)
    t = np.stack([rng.integers(0, E, B), rng.integers(0, R, B), rng.integers(0, E, B)], 1).astype(np.int32)
    triples = torch.as_tensor(t).cuda()
    q, off, ids = k_vs_all_queries(FilterIndex(t, E), t, "o")
    n_q = min(B, len(q))  # the first B distinct (s, p) queries
    q, off, ids = (torch.as_tensor(x).cuda().contiguous() for x in (q[:n_q], off[:n_q + 1], ids))
    engines = {}
    for name, loss in (("one_vs_all", "multiclass_nll"), ("k_vs_all", "nll")):
        eng = KGEEngine("ComplEx", K_USER, 1, E, R, loss=loss, optimizer="sgd")
        eng.init_glorot_uniform(seed=1)
        engines[name] = eng
    steps = {"one_vs_all": lambda eng, s: eng.one_vs_all_backward(triples, "s,o", step=s),
             "k_vs_all": lambda eng, s: eng.k_vs_all_backward(q, "o", off, ids, 0.0, step=s)}
    result = {"gpu": info, "shape": {"n_ent": E, "n_rel": R, "k": K_USER, "B": B, "model": "ComplEx"},
              "dropout": DROPOUT}
    for name, eng in engines.items():
        counter = [0]

        def step():
            counter[0] += 1
            steps[name](eng, counter[0])
        times = {"off": [], "on": []}
        for setting in ("off", "on"):  # warm-up: modules, workspace, both settings
            eng.set_embedding_dropout(*(DROPOUT if setting == "on" else (0.0, 0.0)), seed=3)
            for _ in range(3):
                step()
        for _ in range(a.rounds):
            for setting in ("off", "on"):
                eng.set_embedding_dropout(*(DROPOUT if setting == "on" else (0.0, 0.0)), seed=3)
                times[setting].append(measure.window_ms(step, a.iters, 0))
        off_ms, on_ms = float(np.median(times["off"])), float(np.median(times["on"]))
        # the dropout kernels' own time, profiled in a pass of its own
        eng.set_embedding_dropout(*DROPOUT, seed=3)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.iters):
                step()
            torch.cuda.synchronize()
        kern = {}
        for ev in prof.key_averages():
            if "dropout" in ev.key or "Memset" in ev.key:
                us = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
                kern[ev.key[:80]] = us / a.iters / 1000.0
        eng.set_embedding_dropout(0.0, 0.0)
        result[name] = {"step_ms_off": off_ms, "step_ms_on": on_ms, "overhead_pct": 100.0 * (on_ms / off_ms - 1.0),
                        "rounds_off": times["off"], "rounds_on": times["on"], "dropout_kernels_ms_per_step": kern}
        print("%-10s  off %.3f ms  on %.3f ms  overhead %+.1f %%  dropout kernels %s"
              % (name, off_ms, on_ms, result[name]["overhead_pct"],
                 ", ".join("%s %.3f ms" % kv for kv in kern.items())))
    for eng in engines.values():
        eng.close()
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
