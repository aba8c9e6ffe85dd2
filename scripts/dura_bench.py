#!/usr/bin/env python
"""DURA regulariser benchmark (development aid): times kge_dura_step (csrc/kge_reg_dura.cu) alone, its share of the
steps it is added to, and a torch restatement of the same penalty.

- kge_dura_step alone at cfg2 (ComplEx k = 200, 14,505 entities, 237 relations, B = 27,212), at the 1vsAll FB15k-237
  shape (14,541 entities, B = 1,000) and at 10^6 entities (B = 27,212): CUDA events around the call, median of --iters
  after warm-up.  The bytes it must move: per positive, three row reads (h, r, t) and three row REDs (1,600 B each at
  k = 200) and the 12-byte triple; GB/s is those bytes over the median time.
- The full sampled deferred step of cfg2 (forward_backward(defer=True) + apply_gradients, Adam, self_adversarial) and
  the full 1vsAll "s,o" step at B = 1,000, each with DURA on and off, alternated in one run: --rounds rounds of --iters
  steps each, on and off in turn, the median over all rounds.
- A torch baseline of the same penalty on the same tables at cfg2: gather the rows, the formula, autograd, index_add_
  into the gradients.  Its loss must agree with the kernel's.
Prints the GPU and its power limit first: every number depends on both.

    python scripts/dura_bench.py [--iters N] [--rounds R] [--out FILE.json]
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



W_N, W_P = 1e-3, 1e-3  # lambda 1e-3, alpha = beta = 1
DURA = {"kind": "DURA", "lambda": 1e-3, "alpha": 1.0, "beta": 1.0}


def dura_engine(E, R, B, seed, **kw):
    from ampligraph_b200.engine import KGEEngine
    eng = KGEEngine("ComplEx", 200, kw.pop("eta", 1), E, R, regularizer=[DURA, DURA], **kw)
    eng.init_glorot_uniform(seed=seed)
    return eng, triples(E, R, B, seed)


def row_bytes(eng):
    return 2 * eng.kp * 4  # both halves of a ComplEx row


def alone(E, R, B, iters):
    eng, t = dura_engine(E, R, B, 1)
    ms = float(np.median(events(lambda: eng.dura_backward(t), iters)))
    moved = B * (6 * row_bytes(eng) + 12)
    eng.close()
    return {"n_ent": E, "n_rel": R, "B": B, "ms": ms, "bytes": moved, "GB_per_s": moved / (ms * 1e-3) / 1e9}


def torch_baseline(iters):
    """The same penalty in torch at cfg2: gather, formula, autograd, index_add_; its loss against the kernel's."""
    E, R, B = 14505, 237, 27212
    eng, t = dura_engine(E, R, B, 1)
    kp = eng.kp
    ti = t.long()

    def sq(x):  # |z_d|^2 of padded ComplEx rows [n, ld]: real half [:kp], imaginary half [kp:2kp]
        return x[:, :kp] ** 2 + x[:, kp:2 * kp] ** 2

    def step():
        h = eng.ent.index_select(0, ti[:, 0]).requires_grad_(True)
        r = eng.rel.index_select(0, ti[:, 1]).requires_grad_(True)
        o = eng.ent.index_select(0, ti[:, 2]).requires_grad_(True)
        s = sq(h) + sq(o)
        loss = (W_N * s + W_P * sq(r) * s).sum()
        loss.backward()
        eng.g_ent.index_add_(0, ti[:, 0], h.grad)
        eng.g_ent.index_add_(0, ti[:, 2], o.grad)
        eng.g_rel.index_add_(0, ti[:, 1], r.grad)
        return loss.detach()
    ms = float(np.median(events(step, iters)))
    eng._gblock.zero_()
    eng.loss_acc.zero_()
    want = float(step())
    eng.dura_backward(t)
    got = float(eng.loss_acc[1])
    eng.close()
    assert abs(got - want) <= 1e-5 * abs(want), (got, want)
    return {"B": B, "ms": ms, "loss_torch": want, "loss_kernel": got}


def alternated(kind, rounds, iters):
    """Median step time with DURA off and on, alternated round by round on one engine."""
    from ampligraph_b200.engine import KGEEngine
    if kind == "sampled":
        E, R, B = 14505, 237, 27212
        eng = KGEEngine("ComplEx", 200, 10, E, R, loss="self_adversarial", loss_params=SA, optimizer="adam",
                        regularizer=[DURA, DURA])
    else:
        E, R, B = 14541, 237, 1000
        eng = KGEEngine("ComplEx", 200, 1, E, R, loss="multiclass_nll", optimizer="adam", regularizer=[DURA, DURA])
    eng.init_glorot_uniform(seed=2)
    t = triples(E, R, B, 3)
    eng.set_hot_entities(triples=t)
    state = {"step": 0}

    def step(dura):
        s = state["step"]
        if kind == "sampled":
            eng.forward_backward(t, None, seed=0, step=s, defer=True)
            assert eng._deferred
        else:
            eng.one_vs_all_backward(t, "s,o", step=s)
        if dura:
            eng.dura_backward(t, step=s)
        eng.apply_gradients()
        state["step"] += 1
    res = {"off": [], "on": []}
    for _ in range(rounds):
        for key, dura in (("off", False), ("on", True)):
            res[key] += events(lambda: step(dura), iters, warmup=2)
    eng.close()
    off, on = float(np.median(res["off"])), float(np.median(res["on"]))
    return {"kind": kind, "B": B, "ms_off": off, "ms_on": on, "dura_share_pct": 100.0 * (on - off) / on,
            "spread_off_ms": [float(np.percentile(res["off"], 10)), float(np.percentile(res["off"], 90))],
            "spread_on_ms": [float(np.percentile(res["on"], 10)), float(np.percentile(res["on"], 90))]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dura_bench.py needs a CUDA device: there is no CPU measurement")
    print(gpu_info(), flush=True)
    res = {"gpu": gpu_info(), "alone": [alone(14505, 237, 27212, a.iters), alone(14541, 237, 1000, a.iters),
                                        alone(10 ** 6, 237, 27212, a.iters)],
           "torch_baseline": torch_baseline(a.iters),
           "steps": [alternated("sampled", a.rounds, a.iters), alternated("one_vs_all", a.rounds, a.iters)]}
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
