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
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import measure  # noqa: E402

N3 = {"kind": "N3", "lambda": 1e-3}


def n3_engine(E, R, B, seed, **kw):
    from ampligraph_b200.engine import KGEEngine
    eng = KGEEngine("ComplEx", 200, kw.pop("eta", 1), E, R, regularizer=[N3, N3], **kw)
    eng.init_glorot_uniform(seed=seed)
    return eng, measure.zipf_triples(E, R, B, seed)


def alone(E, R, B, iters):
    eng, t = n3_engine(E, R, B, 1)
    ms = measure.per_call_ms(lambda: eng.n3_backward(t), iters, 3)
    rows = len(torch.unique(torch.cat([t[:, 0], t[:, 2]]))) + len(torch.unique(t[:, 1]))
    out = {"n_ent": E, "n_rel": R, "B": B, "ms": float(np.median(ms)), "distinct_rows": rows,
           # the apply pass reads and writes each distinct row's parameters and gradient (3 x 1600 B); the memset and
           # count pass touch (E + R) x 4 B and B x 12 B
           "GB_per_s": (rows * 3 * 1600 + (E + R) * 4 + B * 12) / (float(np.median(ms)) * 1e-3) / 1e9}
    eng.close()
    return out


def steps(kind, rounds, iters):
    res = measure.regularizer_steps(kind, [N3, N3], lambda eng, t, s: eng.n3_backward(t, step=s), rounds, iters)
    return dict(res, n3_share_pct=100.0 * (res["ms_on"] - res["ms_off"]) / res["ms_on"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("n3_bench.py needs a CUDA device: there is no CPU measurement")
    res = {"gpu": measure.card(), "alone": [alone(14505, 237, 27212, a.iters), alone(14541, 237, 1000, a.iters),
                                            alone(10 ** 6, 237, 27212, a.iters)],
           "steps": [steps("sampled", a.rounds, a.iters), steps("one_vs_all", a.rounds, a.iters)]}
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
