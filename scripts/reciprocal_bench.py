#!/usr/bin/env python
"""Reciprocal-relations benchmark (development aid; DESIGN.md 3.17 and 5) on the FB15k-237 shape: 14,541 entities,
237 relations, ComplEx k = 200.

- Step: a reciprocal 1vsAll 's,o' step, one side-o kge_one_vs_all_step call over the batch's 2B forward and inverse
  rows (2R relation rows), against the plain 's,o' step, one call that runs both sides over the B rows (R relation
  rows), at B = 256, 1,000 and 4,096.  CUDA events around the call, median of --iters after warm-up, the two
  alternated call by call.
- evaluate: filtered evaluate(corrupt_side='s,o') of 20,466 test-shaped triples, filtered by 272,115 training-shaped
  triples, on a reciprocal model against a plain model with the same entity table.  Host clock around the call (it
  ends in a device-to-host copy), median of --eval-iters, alternated.

The kernels are the same, so the expectation is parity within noise.  Prints the GPU and its power limit first: every
number depends on both.

    python scripts/reciprocal_bench.py [--iters N] [--eval-iters N] [--out FILE.json]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import measure  # noqa: E402

E, R, K_USER = 14541, 237, 200  # FB15k-237, ComplEx k = 200
N_TRAIN, N_TEST = 272115, 20466


def triples(rng, n):
    return np.stack([rng.integers(0, E, n), rng.integers(0, R, n), rng.integers(0, E, n)], 1).astype(np.int32)


def step_run(B, iters):
    from ampligraph_b200.datasets import reciprocal_triples
    from ampligraph_b200.engine import KGEEngine
    rng = np.random.default_rng(B)
    K = 2 * K_USER
    ent = rng.uniform(-0.1, 0.1, (E, K)).astype(np.float32)
    rel = rng.uniform(-0.1, 0.1, (2 * R, K)).astype(np.float32)
    X = triples(rng, B)
    plain_rows = torch.as_tensor(X).cuda()
    recip_rows = torch.as_tensor(reciprocal_triples(X, R, "s,o")).cuda()
    plain = KGEEngine("ComplEx", K_USER, 1, E, R, loss="multiclass_nll", optimizer="sgd")
    plain.set_embeddings(ent, rel[:R])
    recip = KGEEngine("ComplEx", K_USER, 1, E, 2 * R, loss="multiclass_nll", optimizer="sgd")
    recip.set_embeddings(ent, rel)
    ms = measure.alternated({"reciprocal": lambda: recip.one_vs_all_backward(recip_rows, "o"),
                             "plain": lambda: plain.one_vs_all_backward(plain_rows, "s,o")}, iters, 1, 3)
    ms_recip, ms_plain = float(np.median(ms["reciprocal"])), float(np.median(ms["plain"]))
    plain.close()
    recip.close()
    res = {"B": B, "reciprocal_ms": ms_recip, "plain_ms": ms_plain, "ratio": ms_recip / ms_plain}
    print("1vsAll 's,o' step B=%-5d  reciprocal (one side-o call, 2B rows) %8.3f ms  plain (one call, both sides) "
          "%8.3f ms  ratio %.3f" % (B, ms_recip, ms_plain, res["ratio"]), flush=True)
    return res


def eval_run(iters):
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    rng = np.random.default_rng(1)
    K = 2 * K_USER
    ent = rng.uniform(-0.1, 0.1, (E, K)).astype(np.float32)
    rel = rng.uniform(-0.1, 0.1, (2 * R, K)).astype(np.float32)
    train, test = triples(rng, N_TRAIN), triples(rng, N_TEST)
    models = {}
    for name, recip in (("reciprocal", True), ("plain", False)):
        m = ScoringBasedEmbeddingModel(eta=1, k=K_USER, scoring_type="ComplEx", max_ent_size=E, max_rel_size=R,
                                       reciprocal_relations=recip)
        m.data_indexer = False
        m.compile(optimizer="adam", loss="multiclass_nll",
                  entity_relation_initializer=[ent, rel if recip else rel[:R]])
        m._build_engine()
        m.is_fitted = True
        models[name] = m
    findex = models["plain"]._build_filter(True, lambda: np.concatenate([train, test]))

    def call(m):
        return m.evaluate(test, corrupt_side="s,o", verbose=False, use_filter=True, _filter_index=findex)
    ranks = {name: call(m) for name, m in models.items()}  # warm-up
    ms = {name: [] for name in models}
    for _ in range(iters):
        for name, m in models.items():
            t0 = time.perf_counter()
            call(m)
            ms[name].append(1e3 * (time.perf_counter() - t0))
    res = {name: float(np.median(v)) for name, v in ms.items()}
    res["ratio"] = res["reciprocal"] / res["plain"]
    # side o uses the same forward rows in both models, so its ranks must agree exactly
    res["side_o_ranks_equal"] = bool(np.array_equal(ranks["reciprocal"][:, 1], ranks["plain"][:, 1]))
    print("filtered evaluate('s,o') of %d triples  reciprocal %8.1f ms  plain %8.1f ms  ratio %.3f  side-o ranks "
          "equal: %s" % (N_TEST, res["reciprocal"], res["plain"], res["ratio"], res["side_o_ranks_equal"]), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--eval-iters", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("reciprocal_bench.py needs a GPU: times are measured on the device, never estimated")
    info = measure.card()
    print(info, flush=True)
    results = {"gpu": info, "steps": [step_run(B, args.iters) for B in (256, 1000, 4096)],
               "evaluate": eval_run(args.eval_iters)}
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
