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
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import measure  # noqa: E402


W_N, W_P = 1e-3, 1e-3  # lambda 1e-3, alpha = beta = 1
DURA = {"kind": "DURA", "lambda": 1e-3, "alpha": 1.0, "beta": 1.0}


def dura_engine(E, R, B, seed, **kw):
    from ampligraph_b200.engine import KGEEngine
    eng = KGEEngine("ComplEx", 200, kw.pop("eta", 1), E, R, regularizer=[DURA, DURA], **kw)
    eng.init_glorot_uniform(seed=seed)
    return eng, measure.zipf_triples(E, R, B, seed)


def row_bytes(eng):
    return 2 * eng.kp * 4  # both halves of a ComplEx row


def alone(E, R, B, iters):
    eng, t = dura_engine(E, R, B, 1)
    ms = float(np.median(measure.per_call_ms(lambda: eng.dura_backward(t), iters, 3)))
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
    ms = float(np.median(measure.per_call_ms(step, iters, 3)))
    eng._gblock.zero_()
    eng.loss_acc.zero_()
    want = float(step())
    eng.dura_backward(t)
    got = float(eng.loss_acc[1])
    eng.close()
    assert abs(got - want) <= 1e-5 * abs(want), (got, want)
    return {"B": B, "ms": ms, "loss_torch": want, "loss_kernel": got}


def steps(kind, rounds, iters):
    res = measure.regularizer_steps(kind, [DURA, DURA], lambda eng, t, s: eng.dura_backward(t, step=s), rounds, iters)
    return dict(res, dura_share_pct=100.0 * (res["ms_on"] - res["ms_off"]) / res["ms_on"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dura_bench.py needs a CUDA device: there is no CPU measurement")
    print(measure.card(), flush=True)
    res = {"gpu": measure.card(), "alone": [alone(14505, 237, 27212, a.iters), alone(14541, 237, 1000, a.iters),
                                            alone(10 ** 6, 237, 27212, a.iters)],
           "torch_baseline": torch_baseline(a.iters),
           "steps": [steps("sampled", a.rounds, a.iters), steps("one_vs_all", a.rounds, a.iters)]}
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
