#!/usr/bin/env python
"""Shared-negatives benchmark (development aid; DESIGN.md 3.21, 5): kge_shared_negatives_step against the per-positive
fused step (kge_train_step, in-kernel draws) at the same eta, on one GPU, with Zipf positives:
  rotate   RotatE k = 1,000, eta = 256, B = 1,024, self_adversarial, FB15k-237's shape (14,541 entities, 237 relations)
  transe   TransE k = 1,000, eta = 256, B = 1,024, the same shape
  complex  ComplEx k = 200, eta = 256, B = 27,212, cfg2's shape (14,505 entities, 237 relations)

For each shape: the step's device time (forward + backward into the gradient tables, no optimizer; CUDA events around
each call, median of the alternated rounds) of the fused step and of the shared step at C = 16, 64 and 256; triples/s;
and the candidate-row bytes per step computed from the shapes (per-positive: B eta rows; shared: per chunk slice of 16
positives, eta rows) with the achieved rate against 3.35 TB/s.  Prints the GPU and its power limit first.

    python scripts/shared_negatives_bench.py [--iters N] [--rounds R] [--out FILE.json]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import measure  # noqa: E402

SHAPES = {
    "rotate": dict(model="RotatE", k=1000, eta=256, B=1024, E=14541, R=237, loss="self_adversarial",
                   lp={"margin": 9.0, "alpha": 1.0}),
    "transe": dict(model="TransE", k=1000, eta=256, B=1024, E=14541, R=237, loss="self_adversarial",
                   lp={"margin": 9.0, "alpha": 1.0}),
    "complex": dict(model="ComplEx", k=200, eta=256, B=27212, E=14505, R=237, loss="multiclass_nll", lp={}),
}
CHUNKS = (16, 64, 256)
PEAK = 3.35e12
SLICE = 16  # positives per CTA of the shared step's passes (kge_train_shared.cu: SN_PS)


def run(name, s, a):
    from ampligraph_b200.engine import KGEEngine
    eng = KGEEngine(s["model"], s["k"], s["eta"], s["E"], s["R"], loss=s["loss"], loss_params=s["lp"])
    eng.init_glorot_uniform(seed=1)
    t = measure.zipf_triples(s["E"], s["R"], s["B"], seed=2)
    B, eta, row = s["B"], s["eta"], 4 * eng.ld

    def zero():
        eng.g_ent.zero_()
        eng.g_rel.zero_()

    fns = {"fused": lambda: eng.forward_backward(t, None, seed=3, step=1)}
    for C in CHUNKS:
        fns["C=%d" % C] = (lambda C=C: eng.shared_negatives_backward(t, C, seed=3, step=1))
    ms = measure.alternated(fns, a.rounds, a.iters, 3)
    zero()
    out = {}
    for key, v in ms.items():
        med = sorted(v)[len(v) // 2]
        if key == "fused":
            rows = B * eta
        else:
            C = int(key[2:])
            slices = sum(-(-min(C, B - c0) // SLICE) for c0 in range(0, B, C))
            rows = slices * eta
        out[key] = dict(ms=med, triples_per_s=B / med * 1e3, cand_bytes=rows * row,
                        cand_rate=rows * row / (med * 1e-3), cand_share_of_peak=rows * row / (med * 1e-3) / PEAK)
        print("%-8s %-6s %8.3f ms  %10.0f triples/s  cand rows %8.1f MB  %7.1f GB/s (%.1f%% of 3.35 TB/s)"
              % (name, key, med, out[key]["triples_per_s"], rows * row / 1e6, out[key]["cand_rate"] / 1e9,
                 100 * out[key]["cand_share_of_peak"]), flush=True)
    eng.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    print(measure.card(), flush=True)
    res = {"card": measure.card()}
    for name in a.shapes.split(","):
        res[name] = run(name, SHAPES[name], a)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
