"""Time the optimizer kernels per kind on bench.py's cfg2 parameter block: the [ent | rel] block of ComplEx k=200 (14,505 +
237 rows, ld 400), CUDA events around each call.

  kge_optimizer_step           the dense rule over the whole block (one launch)
  kge_optimizer_step_deferred  the owner-per-row kernel: a deferred step's replaced-row sum + the dense rule
                               (27,212 Zipf positives, eta 10, as bench.py), timed alone
  kge_optimizer_step_decay     Nadam's IndexedSlices rule over the whole block with half of the rows stamped: the
                               unstamped half moves only m and v (4 streams, plus the row stamps)

Achieved GB/s counts the algorithmic streams of the dense rule, from shapes: per element the parameter and the gradient
(read, then written / zeroed) and every slot the kind uses (read and written) -- 6 fp32 streams for one-slot RMSprop, 8 for
the two-slot kinds (Nadam and Ftrl among them) and Adam.  The owner kernel also reads the bucket entries and their rows; its GB/s counts the same
streams, so it understates that kernel's traffic.

  python scripts/optim_bench.py [--iters 200] [--warmup 20]
Prints the card and its power limit, then one JSON line per (kernel, kind)."""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import measure  # noqa: E402
from ampligraph_b200 import _lib  # noqa: E402
from ampligraph_b200.engine import KGEEngine, optimizer_slots  # noqa: E402

KINDS = [("adam", {}), ("rmsprop", {}), ("rmsprop", {"centered": True}), ("rmsprop", {"momentum": 0.9}),
         ("adadelta", {"learning_rate": 1.0}), ("adamax", {}), ("nadam", {}), ("ftrl", {}),
         ("ftrl", {"learning_rate_power": -0.25})]
E, R, K, ETA, B = 14505, 237, 200, 10, 27212


def zipf_triples(n, rng):
    w = 1.0 / np.arange(1, E + 1)
    cdf = np.cumsum(w / w.sum())
    perm = rng.permutation(E)
    s, o = perm[np.searchsorted(cdf, rng.random(n))], perm[np.searchsorted(cdf, rng.random(n))]
    return np.stack([s, rng.integers(0, R, n), o], 1).astype(np.int32)


def time_calls(call, before, iters, warmup):
    """mean device time of call() in microseconds, with before() run outside each timed call.  before() queues GPU work
    (a training step), so the timed call's launch waits on the stream rather than on the host."""
    for _ in range(warmup):
        before()
        call()
    torch.cuda.synchronize()
    marks = []
    for _ in range(iters):
        before()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        call()
        b.record()
        marks.append((a, b))
    torch.cuda.synchronize()
    return 1e3 * sum(a.elapsed_time(b) for a, b in marks) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("optim_bench.py needs a CUDA device")
    print(measure.card())
    rng = np.random.default_rng(0)
    t = torch.as_tensor(zipf_triples(B, rng)).cuda()
    for name, params in KINDS:
        eng = KGEEngine("ComplEx", K, ETA, E, R, loss="self_adversarial", optimizer=name,
                        optimizer_params=dict({"learning_rate": 1e-3}, **params))
        eng.init_glorot_uniform(1)
        rows, ld = E + R, eng.ld
        streams = 4 + 2 * sum(v is not None for v in optimizer_slots(eng.opt_cfg))
        nbytes = rows * ld * 4 * streams
        label = name + "".join("_%s" % k for k in params if k != "learning_rate")

        ptr = lambda x: C.c_void_p(x.data_ptr()) if x is not None else None

        def dense():
            eng.begin_step()
            _lib.check(eng.lib.kge_optimizer_step(eng.h, C.byref(eng.opt_cfg), eng.t, ptr(eng._pblock), ptr(eng._gblock),
                                                  ptr(eng._sblocks[0]), ptr(eng._sblocks[1]), rows, None, eng._stream()))
        us = 1e3 * measure.window_ms(dense, args.iters, args.warmup)
        print(json.dumps({"kernel": "kge_optimizer_step", "kind": label, "us": round(us, 2), "streams": streams,
                          "GB_per_s": round(nbytes / us / 1e3, 1)}))

        step = [0]

        def pend():
            eng.forward_backward(t, None, seed=1, step=step[0], defer=True)
            step[0] += 1
            assert eng._deferred

        us = time_calls(eng.apply_gradients, pend, args.iters, args.warmup)
        print(json.dumps({"kernel": "kge_optimizer_step_deferred", "kind": label, "us": round(us, 2), "streams": streams,
                          "GB_per_s": round(nbytes / us / 1e3, 1)}))
        if name == "nadam":
            stamps = torch.as_tensor(np.where(rng.random(rows) < 0.5, 1, 0).astype(np.int32)).cuda()

            def decay():
                eng.begin_step()
                _lib.check(eng.lib.kge_optimizer_step_decay(eng.h, C.byref(eng.opt_cfg), eng.t, ptr(eng._pblock),
                                                            ptr(eng._gblock), ptr(eng._sblocks[0]), ptr(eng._sblocks[1]),
                                                            rows, ptr(stamps), 1, eng._stream()))
            us = 1e3 * measure.window_ms(decay, args.iters, args.warmup)
            dbytes = rows * ld * 4 * 6 + rows * 4  # half the rows 8 streams, half 4, and the stamps
            print(json.dumps({"kernel": "kge_optimizer_step_decay", "kind": label, "us": round(us, 2), "streams": 6,
                              "GB_per_s": round(dbytes / us / 1e3, 1)}))
        eng.close()


if __name__ == "__main__":
    main()
