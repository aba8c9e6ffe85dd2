#!/usr/bin/env python
"""N3 regulariser benchmark (development aid): times kge_n3_step (csrc/kge_reg_n3.cu) alone and its share of the steps
it is added to.

- kge_n3_step alone at cfg2 (ComplEx k = 200, 14,505 entities, 237 relations, B = 27,212), at the 1vsAll FB15k-237
  shape (14,541 entities, B = 1,000) and at 10^6 entities (B = 27,212): CUDA events around the call, median of --iters
  after warm-up.  The count pass reads B triples; the apply pass reads and writes the distinct rows the batch uses.
- The full sampled deferred step of cfg2 (forward_backward(defer=True) + apply_gradients, Adam, self_adversarial) and
  the full 1vsAll "s,o" step at B = 1,000, each with N3 on and off, alternated in one run: --rounds rounds of --iters
  steps each, on and off in turn, the median over all rounds.
Prints the GPU and its power limit first: every number depends on both.

    python scripts/n3_bench.py [--iters N] [--rounds R] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SA = {"margin": 3.0, "alpha": 0.5}


def gpu_info():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                            stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True).stdout.strip()
    except OSError:
        pl = "unknown"
    return "%s, power limit / max SM clock: %s" % (name, pl)


def events(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return ms


def triples(E, R, B, seed):
    rng = np.random.default_rng(seed)
    # Zipf(1.0) entities, as bench.py's synthetic KG: frequent entities repeat within a batch
    w = 1.0 / np.arange(1, E + 1)
    p = w / w.sum()
    t = np.stack([rng.choice(E, B, p=p), rng.integers(0, R, B), rng.choice(E, B, p=p)], 1)
    return torch.as_tensor(t.astype(np.int32)).cuda().contiguous()


def n3_engine(E, R, B, seed, **kw):
    from ampligraph_b200.engine import KGEEngine
    eng = KGEEngine("ComplEx", 200, kw.pop("eta", 1), E, R,
                    regularizer=[{"kind": "N3", "lambda": 1e-3}, {"kind": "N3", "lambda": 1e-3}], **kw)
    eng.init_glorot_uniform(seed=seed)
    return eng, triples(E, R, B, seed)


def alone(E, R, B, iters):
    eng, t = n3_engine(E, R, B, 1)
    ms = events(lambda: eng.n3_backward(t), iters)
    rows = len(torch.unique(torch.cat([t[:, 0], t[:, 2]]))) + len(torch.unique(t[:, 1]))
    out = {"n_ent": E, "n_rel": R, "B": B, "ms": float(np.median(ms)), "distinct_rows": rows,
           # the apply pass reads and writes each distinct row's parameters and gradient (3 x 1600 B); the memset and
           # count pass touch (E + R) x 4 B and B x 12 B
           "GB_per_s": (rows * 3 * 1600 + (E + R) * 4 + B * 12) / (float(np.median(ms)) * 1e-3) / 1e9}
    eng.close()
    return out


def alternated(kind, rounds, iters):
    """Median step time with N3 off and on, alternated round by round on one engine."""
    from ampligraph_b200.engine import KGEEngine
    if kind == "sampled":
        E, R, B = 14505, 237, 27212
        eng = KGEEngine("ComplEx", 200, 10, E, R, loss="self_adversarial", loss_params=SA, optimizer="adam",
                        regularizer=[{"kind": "N3", "lambda": 1e-3}, {"kind": "N3", "lambda": 1e-3}])
    else:
        E, R, B = 14541, 237, 1000
        eng = KGEEngine("ComplEx", 200, 1, E, R, loss="multiclass_nll", optimizer="adam",
                        regularizer=[{"kind": "N3", "lambda": 1e-3}, {"kind": "N3", "lambda": 1e-3}])
    eng.init_glorot_uniform(seed=2)
    t = triples(E, R, B, 3)
    eng.set_hot_entities(triples=t)
    state = {"step": 0}

    def step(n3):
        s = state["step"]
        if kind == "sampled":
            eng.forward_backward(t, None, seed=0, step=s, defer=True)
            assert eng._deferred
        else:
            eng.one_vs_all_backward(t, "s,o", step=s)
        if n3:
            eng.n3_backward(t, step=s)
        eng.apply_gradients()
        state["step"] += 1
    res = {"off": [], "on": []}
    for _ in range(rounds):
        for key, n3 in (("off", False), ("on", True)):
            res[key] += events(lambda: step(n3), iters, warmup=2)
    eng.close()
    off, on = float(np.median(res["off"])), float(np.median(res["on"]))
    return {"kind": kind, "B": B, "ms_off": off, "ms_on": on, "n3_share_pct": 100.0 * (on - off) / on,
            "spread_off_ms": [float(np.percentile(res["off"], 10)), float(np.percentile(res["off"], 90))],
            "spread_on_ms": [float(np.percentile(res["on"], 10)), float(np.percentile(res["on"], 90))]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("n3_bench.py needs a CUDA device: there is no CPU measurement")
    res = {"gpu": gpu_info(), "alone": [alone(14505, 237, 27212, a.iters), alone(14541, 237, 1000, a.iters),
                                        alone(10 ** 6, 237, 27212, a.iters)],
           "steps": [alternated("sampled", a.rounds, a.iters), alternated("one_vs_all", a.rounds, a.iters)]}
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
