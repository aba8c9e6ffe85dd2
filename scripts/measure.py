"""Measurement shared by the benchmark scripts.

Every time a script reports depends on the card and its power limit, so each one prints card() in the same run.  Every
timed callable is warmed up first, and CUDA events are recorded around work that ends in a synchronise."""
import subprocess

import numpy as np
import torch


def card():
    """The GPU's name, its power limit and its max SM clock."""
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                            stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True).stdout.strip()
    except OSError:
        pl = "unknown"
    return "%s, power limit / max SM clock: %s" % (name, pl)


def per_call_ms(fn, iters, warmup, before=None):
    """The device time in ms of each of `iters` calls of fn() after `warmup` untimed ones: an event pair around each
    call and a synchronise after it.  before(), if given, runs untimed ahead of each timed call (an L2 flush, say)."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(iters):
        if before is not None:
            before()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return ms


def window_ms(fn, iters, warmup):
    """The mean device time in ms per call of `iters` back-to-back calls of fn() between two events, after `warmup`
    untimed calls."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def alternated(fns, rounds, iters, warmup):
    """{name: per-call ms} of the callables in `fns` ({name: callable}), interleaved so that the shared machine's drift
    hits them alike: `warmup` untimed calls of each in turn, then `rounds` rounds in which each makes `iters` timed
    calls (per_call_ms) in turn."""
    for _ in range(warmup):
        for fn in fns.values():
            fn()
    ms = {name: [] for name in fns}
    for _ in range(rounds):
        for name, fn in fns.items():
            ms[name] += per_call_ms(fn, iters, 0)
    return ms


def zipf_triples(E, R, B, seed):
    """B device triples [B, 3] int32: Zipf(1.0) subjects and objects, as bench.py's synthetic KG, so that frequent
    entities repeat within a batch; uniform relations."""
    rng = np.random.default_rng(seed)
    w = 1.0 / np.arange(1, E + 1)
    p = w / w.sum()
    t = np.stack([rng.choice(E, B, p=p), rng.integers(0, R, B), rng.choice(E, B, p=p)], 1)
    return torch.as_tensor(t.astype(np.int32)).cuda().contiguous()


def regularizer_steps(kind, regularizer, backward, rounds, iters):
    """Step times with a regulariser off and on, alternated round by round on one ComplEx k = 200 engine with Adam.
    kind "sampled": cfg2's deferred step (forward_backward(defer=True) + apply_gradients, self-adversarial, eta 10,
    14,505 entities, 237 relations, B = 27,212); kind "one_vs_all": the 1vsAll "s,o" step on the FB15k-237 shape
    (14,541 entities, B = 1,000).  `regularizer` is the engine's regularizer argument; backward(eng, t, step) adds the
    regulariser's gradient of the step's triples.  -> medians and 10th / 90th percentiles of both settings."""
    from ampligraph_b200.engine import KGEEngine
    if kind == "sampled":
        E, R, B = 14505, 237, 27212
        eng = KGEEngine("ComplEx", 200, 10, E, R, loss="self_adversarial",
                        loss_params={"margin": 3.0, "alpha": 0.5}, optimizer="adam", regularizer=regularizer)
    else:
        E, R, B = 14541, 237, 1000
        eng = KGEEngine("ComplEx", 200, 1, E, R, loss="multiclass_nll", optimizer="adam", regularizer=regularizer)
    eng.init_glorot_uniform(seed=2)
    t = zipf_triples(E, R, B, 3)
    eng.set_hot_entities(triples=t)
    state = {"step": 0}

    def step(on):
        s = state["step"]
        if kind == "sampled":
            eng.forward_backward(t, None, seed=0, step=s, defer=True)
            assert eng._deferred
        else:
            eng.one_vs_all_backward(t, "s,o", step=s)
        if on:
            backward(eng, t, s)
        eng.apply_gradients()
        state["step"] += 1
    res = alternated({"off": lambda: step(False), "on": lambda: step(True)}, rounds, iters, 2)
    eng.close()
    return {"kind": kind, "B": B, "ms_off": float(np.median(res["off"])), "ms_on": float(np.median(res["on"])),
            "spread_off_ms": [float(np.percentile(res["off"], 10)), float(np.percentile(res["off"], 90))],
            "spread_on_ms": [float(np.percentile(res["on"], 10)), float(np.percentile(res["on"], 90))]}
