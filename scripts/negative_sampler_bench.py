#!/usr/bin/env python
"""Negative sampler benchmark (development aid; DESIGN.md 3.18, 5): kge_sample_negatives (csrc/kge_negatives.cu) on
bench.py's workload, BASELINE.json configs[1]: ComplEx k = 200, eta = 10, B = 27,212, the seeded FB15k-237-shaped
synthetic KG of bench.py (14,505 entities, 237 relations, 272,115 triples), fit's 10 filter attempts.

- The sampler kernel alone per mode (uniform, bernoulli, pseudo_typed, each without and with the filter): its device
  time from torch.profiler over --iters calls, and CUDA events around one call (which include the host's issue of
  it), medians; steps varied so every call draws afresh.
- The full deferred step (forward_backward(defer=True) + apply_gradients, Adam, self_adversarial) with in-kernel
  Philox draws, with injected uniform or pseudo-typed corruptions drawn beforehand, and with the sampler's launch
  inside the step for each mode; alternated in one run, --rounds rounds of --iters steps each, the median over all
  rounds.
- The share of emitted corruptions that are training triples per mode, over --share-steps batches (with the filter:
  the misses).
Prints the GPU and its power limit first: every number depends on both.

    python scripts/negative_sampler_bench.py [--iters N] [--rounds R] [--out FILE.json]
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

MODES = [(s, f) for s in ("uniform", "bernoulli", "pseudo_typed") for f in (False, True)]
ATTEMPTS = 10  # models.NEGATIVE_FILTER_ATTEMPTS


def name(mode):
    return mode[0] + ("+filter" if mode[1] else "")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--share-steps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("negative_sampler_bench.py needs a CUDA device: there is no CPU measurement")
    import bench
    from ampligraph_b200.datasets import negative_sampler_tables
    from ampligraph_b200.engine import KGEEngine, NegativeSamplerTables
    print(measure.card(), flush=True)
    c = bench.CFG
    E, R, B, eta = c["n_ent"], c["n_rel"], c["batch"], c["eta"]
    kg = bench.synthetic_kg(E, R, c["n_triples"])
    eng = KGEEngine(c["model"], c["k"], eta, E, R, loss=c["loss"], loss_params=c["loss_params"], optimizer="adam",
                    optimizer_params={"learning_rate": c["lr"]})
    eng.init_glorot_uniform(seed=1)
    eng.set_hot_entities(triples=kg)
    data = torch.as_tensor(kg).cuda().contiguous()
    batch = data[:B]
    tables = {}
    for mode in MODES:
        host = negative_sampler_tables(kg, E, R, mode[0], mode[1])
        tables[mode] = NegativeSamplerTables(host, ATTEMPTS, eng.device)
    res = {"gpu": measure.card(), "workload": "cfg2: ComplEx k=200, eta=10, B=27,212, FB15k-237-shaped synthetic KG",
           "kernel_us": {}, "step_ms": {}, "known_share": {}}

    # the kernel alone: its device time from torch.profiler (CUDA events around one call would also time the host's
    # issue of it, which is longer than the kernel), and the call with events for comparison
    from torch.profiler import ProfilerActivity, profile
    for mode in MODES:
        state = {"step": 0}

        def call():
            eng.sample_negatives(batch, tables[mode], 0, state["step"])
            state["step"] += 1
        call_ms = measure.per_call_ms(call, a.iters, 3)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.iters):
                call()
            torch.cuda.synchronize()
        us = [e.time_range.elapsed_us() for e in prof.events() if "kge_negatives_kernel" in e.name]
        assert len(us) == a.iters, len(us)
        res["kernel_us"][name(mode)] = {"kernel_median": float(np.median(us)), "kernel_p90": float(np.percentile(us, 90)),
                                        "call_with_issue_median": 1e3 * float(np.median(call_ms))}
        eng.read_negative_misses()
    print(json.dumps(res["kernel_us"]), flush=True)

    # the full step
    injected = tuple(x.clone() for x in eng.sample_negatives(batch, tables[("uniform", False)], 0, 10 ** 6))
    # the pseudo-typed corruptions drawn beforehand: what the training kernels cost on their distribution alone
    injected_pt = tuple(x.clone() for x in eng.sample_negatives(batch, tables[("pseudo_typed", False)], 0, 10 ** 6))
    state = {"step": 0}

    def step(kind):
        s = state["step"]
        if kind == "in-kernel":
            negs = None
        elif kind == "injected":
            negs = injected
        elif kind == "injected pseudo_typed":
            negs = injected_pt
        else:
            negs = eng.sample_negatives(batch, tables[kind], 0, s)
        eng.forward_backward(batch, negs, seed=0, step=s, defer=True)
        assert eng._deferred
        eng.apply_gradients()
        state["step"] += 1
    kinds = ["in-kernel", "injected", "injected pseudo_typed"] + MODES
    times = measure.alternated({str(k): lambda k=k: step(k) for k in kinds}, a.rounds, a.iters, 2)
    for kind in kinds:
        ms = times[str(kind)]
        key = kind if isinstance(kind, str) else "sampler " + name(kind)
        res["step_ms"][key] = {"median": float(np.median(ms)), "p10": float(np.percentile(ms, 10)),
                               "p90": float(np.percentile(ms, 90))}
    eng.read_negative_misses()
    print(json.dumps(res["step_ms"]), flush=True)

    # the share of known triples among the emitted corruptions
    known = np.unique(kg.astype(np.int64) @ np.array([E * R, E, 1], np.int64))
    for mode in MODES:
        hits = total = 0
        for s in range(a.share_steps):
            b = data[(s * B) % len(kg):(s * B) % len(kg) + B]
            repl, keep = eng.sample_negatives(b, tables[mode], 0, s)
            t = b.repeat(eta, 1).long()
            k = keep.bool()
            sub = torch.where(k, t[:, 0], repl.long())
            obj = torch.where(k, repl.long(), t[:, 2])
            code = ((sub * R + t[:, 1]) * E + obj).cpu().numpy()
            hits += int(np.isin(code, known).sum())
            total += code.size
        misses = eng.read_negative_misses()
        res["known_share"][name(mode)] = {"known": hits, "corruptions": total, "share_pct": 100.0 * hits / total,
                                          "counted_misses": misses}
    print(json.dumps(res["known_share"]), flush=True)
    eng.close()
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
