#!/usr/bin/env python
"""Relation-prediction benchmark (development aid): times the relation side (side 'p', csrc/kge_rank_rel.cu) on three
dataset shapes -- FB15k-237, FB15k and YAGO3-10 (entities, relations, test-set size) -- with random tables, against the
baseline a user has without it: tile the b x R completed triples through the kernel model.predict runs
(engine.score) and count the ranks with torch on the GPU.

Reported per shape: the kernel time of one unfiltered kge_rank call over the whole test set and of one kge_topk call
(CUDA events, median of several runs), the end-to-end times of evaluate(corrupt_side='p') unfiltered and filtered and of
query_topn_batch(side='p', top_n=10), the baseline's time (from the same tables), and the achieved fp32 operation rate
of the rank kernel, counted from the shapes by pair_flops() below.  Prints the GPU and its power limit first: every
number depends on both.

    python scripts/relation_bench.py [--models ComplEx,TransE,...] [--iters N]
"""
import argparse
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import measure  # noqa: E402

# (name, entities, relations, test triples)
SHAPES = [("FB15k-237", 14505, 237, 20466), ("FB15k", 14951, 1345, 59071), ("YAGO3-10", 123182, 37, 5000)]


def pair_flops(model, k):
    """fp32 operations of one (query, relation) score of the relation-side chain, an FMA counted as 2 and a square root
    as 1: per column TransE s + p, - o, acc + |.| (3); DistMult s * p, fma (3); per column pair ComplEx / HolE two
    halves of mul + fma + fma (10); RotatE the rotation (2 mul + 2 fma = 6), two differences, the squared modulus
    (mul + fma = 3), sqrt and the sum (13)."""
    return k * {"TransE": 3, "DistMult": 3, "ComplEx": 10, "HolE": 10, "RotatE": 13}[model]


def wall(fn, iters):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def model_for(model, k, E, R):
    """A facade model on random tables, ids as labels (no indexer)."""
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    m = ScoringBasedEmbeddingModel(eta=1, k=k, scoring_type=model, max_ent_size=E, max_rel_size=R, seed=1)
    m.data_indexer = False
    m.compile(optimizer="adam", loss="pairwise")
    m._build_engine()
    m.is_fitted = True
    return m


def baseline_ranks(eng, t, R, chunk=4096):
    """What a user writes without the relation side: every (s, r, o) through predict's kernel, worst-rank counts in torch.
    -> int32 ranks (count + 1)."""
    out = []
    rels = torch.arange(R, dtype=torch.int32, device=t.device)
    for s in range(0, t.shape[0], chunk):
        q = t[s:s + chunk]
        n = q.shape[0]
        full = torch.stack([q[:, 0].repeat_interleave(R), rels.repeat(n), q[:, 2].repeat_interleave(R)], 1).contiguous()
        grid = (eng.score(full) * 1000.0).to(torch.int32).view(n, R)
        pos = (eng.score(q.contiguous()) * 1000.0).to(torch.int32)
        out.append((grid >= pos[:, None]).sum(1).to(torch.int32) + 1)
    return torch.cat(out)


def run(model, k, name, E, R, b, iters):
    from ampligraph_b200.discovery import query_topn_batch
    rng = np.random.default_rng(0)
    m = model_for(model, k, E, R)
    eng = m.engine
    X = np.stack([rng.integers(0, E, b), rng.integers(0, R, b), rng.integers(0, E, b)], 1).astype(np.int32)
    t = torch.as_tensor(X).cuda()
    rank_ms = float(np.median(measure.per_call_ms(lambda: eng.rank(t, "p", "worst"), iters, 1)))
    topk_ms = float(np.median(measure.per_call_ms(lambda: eng.topk(t, "p", 10), iters, 1)))
    base_ms = float(np.median(measure.per_call_ms(lambda: baseline_ranks(eng, t, R), iters, 1)))
    ev_ms = wall(lambda: m.evaluate(X, corrupt_side="p", verbose=False), iters)
    evf_ms = wall(lambda: m.evaluate(X, corrupt_side="p", use_filter={"test": X}, verbose=False), iters)
    q_ms = wall(lambda: query_topn_batch(m, X, side="p", top_n=10), max(1, iters // 2))
    # the baseline and the relation side agree on the unfiltered worst ranks (to fp32 rounding of near-ties)
    same = float((baseline_ranks(eng, t, R).cpu().numpy() == m.evaluate(X, corrupt_side="p", verbose=False)[:, 0]).mean())
    flops = float(b) * R * pair_flops(model, k)
    print("%-9s %-8s k=%-3d E=%-6d R=%-5d b=%-5d  kge_rank %8.2f ms (%6.2f TFLOP/s fp32)  kge_topk(10) %8.2f ms  "
          "baseline predict+torch %9.2f ms (%5.1fx)  evaluate %8.1f ms  evaluate filtered %8.1f ms  "
          "query_topn_batch %8.1f ms  ranks equal to baseline %.4f"
          % (name, model, k, E, R, b, rank_ms, flops / rank_ms * 1e-9, topk_ms, base_ms, base_ms / rank_ms, ev_ms, evf_ms,
             q_ms, same), flush=True)
    eng.close()
    del m, eng, t
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="ComplEx")
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("relation_bench.py needs a GPU: times are measured on the device, never estimated")
    print(measure.card(), flush=True)
    for model in args.models.split(","):
        for name, E, R, b in SHAPES:
            run(model, 200, name, E, R, b, args.iters)


if __name__ == "__main__":
    main()
