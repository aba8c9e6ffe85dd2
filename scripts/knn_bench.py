#!/usr/bin/env python
"""Nearest-neighbour / duplicate-search benchmark (development aid).

  (a) kge_knn, 1,024 queries, top 10, over a cfg2-shaped ComplEx k = 200 entity table (14,505 x 400), both metrics,
      alternated in the same run with kge_topk for TransE k = 400 (the same width; its object side is the L1 chain);
  (b) the nearest-other-row pass of find_duplicates(tolerance='auto') over all 14,505 entities;
  (c) find_duplicates(mode='e', tolerance='auto') end to end on the GPU, and the reference algorithm
      (discovery.py:939-980: spatial.distance_matrix, then optimize.bisect over sklearn radius_neighbors self-joins)
      on the host CPU -- a host number, labelled as such, partly extrapolated (see case_c);
  (d) kge_knn, 1,024 queries against 1,000,000 entities.
CUDA events, L2 flushed between iterations; prints the GPU and its power limit, because every number depends on both."""
import logging
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import measure  # noqa: E402
from ampligraph_b200.engine import KGEEngine  # noqa: E402


def case_a(iters=20, rounds=3):
    rng = np.random.default_rng(0)
    E, b, top, R = 14505, 1024, 10, 237
    cx = KGEEngine("ComplEx", 200, 1, E, R)
    cx.init_glorot_uniform(1)
    te = KGEEngine("TransE", 400, 1, E, R)
    te.init_glorot_uniform(2)
    q = torch.as_tensor(rng.integers(0, E, b).astype(np.int32)).cuda()
    t = torch.as_tensor(np.stack([rng.integers(0, E, b), rng.integers(0, R, b), rng.integers(0, E, b)], 1)
                        .astype(np.int32)).cuda()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    res = {"euclidean": [], "manhattan": [], "topk": []}
    for _ in range(rounds):  # alternated, so that drift of the shared machine hits all three alike
        res["topk"].append(np.median(measure.per_call_ms(lambda: te.topk(t, "o", top), iters, 2, before=flush.zero_)))
        for metric in ("euclidean", "manhattan"):
            res[metric].append(np.median(measure.per_call_ms(lambda: cx.knn(cx.ent, q, top, metric), iters, 2,
                                                             before=flush.zero_)))
    tk = np.median(res["topk"])
    print("(a) E=%d ld=400 b=%d top=%d: kge_topk TransE k=400 side o %.1f us" % (E, b, top, tk * 1e3))
    for metric in ("euclidean", "manhattan"):
        m = np.median(res[metric])
        print("    kge_knn %-9s %.1f us  (%.3f x kge_topk; rounds: %s)"
              % (metric, m * 1e3, m / tk, " ".join("%.1f" % (x * 1e3) for x in res[metric])))
    cx.close()
    te.close()


def case_b(iters=10):
    rng = np.random.default_rng(1)
    E = 14505
    eng = KGEEngine("ComplEx", 200, 1, E, 1)
    eng.init_glorot_uniform(3)
    pts = eng.ent[torch.as_tensor(rng.permutation(E), device="cuda")].contiguous()
    every = torch.arange(E, dtype=torch.int32, device="cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")

    def d1_pass(metric):
        for s in range(0, E, 1024):
            qq = every[s:s + 1024]
            off = torch.arange(qq.numel() + 1, dtype=torch.int64, device="cuda")
            eng.knn(pts, qq, 1, metric, n_cand=E, filt_off=off, filt_idx=qq)
    for metric in ("euclidean", "manhattan"):
        ms = np.median(measure.per_call_ms(lambda: d1_pass(metric), iters, 2, before=flush.zero_))
        print("(b) nearest-other-row pass, %d x 400, %-9s %.2f ms" % (E, metric, ms))
    eng.close()


def case_c(budget=200.0):
    from scipy import optimize, spatial
    from sklearn.neighbors import NearestNeighbors
    from ampligraph_b200.discovery import find_duplicates
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    rng = np.random.default_rng(2)
    E, R, n = 14505, 237, 100_000
    t = np.stack([rng.integers(0, E, n), rng.integers(0, R, n), rng.integers(0, E, n)], 1)
    t[:E, 0] = np.arange(E)  # every entity appears
    X = np.stack([np.char.add("e", t[:, 0].astype(str)), np.char.add("r", t[:, 1].astype(str)),
                  np.char.add("e", t[:, 2].astype(str))], 1)
    m = ScoringBasedEmbeddingModel(eta=5, k=200, scoring_type="ComplEx", seed=0)
    m.compile(optimizer="adam", loss="multiclass_nll")
    m.fit(X, batch_size=10000, epochs=1, verbose=False)
    ents = np.unique(X[:, 0])
    find_duplicates(ents, m, tolerance="auto")  # warm-up
    evals = []  # bisection steps, counted from the verbose log
    counter = logging.Handler()
    counter.emit = lambda rec: evals.append(rec)
    log = logging.getLogger("ampligraph_b200.discovery")
    log.addHandler(counter)
    log.setLevel(logging.INFO)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    dups, tol = find_duplicates(ents, m, tolerance="auto", verbose=True)
    torch.cuda.synchronize()
    gpu_s = time.perf_counter() - t0
    log.removeHandler(counter)
    print("(c) find_duplicates(mode='e', tolerance='auto'), %d entities x 400: GPU end to end %.3f s (tolerance %.6f, "
          "%d groups, %d bisection steps)" % (len(ents), gpu_s, tol, len(dups), len(evals)), flush=True)

    # The reference (discovery.py:922-980) verbatim on the host; each bisection step is a radius_neighbors self-join.
    # It runs until `budget` seconds have passed, then the total is extrapolated from the measured steps and the number
    # of steps the same bisection took above.
    emb = m.get_embeddings(ents, embedding_type="e")
    steps = []

    class Budget(Exception):
        pass

    def get_dups(tol):  # discovery.py:922-951
        nn = NearestNeighbors(metric="l2", radius=tol)
        nn.fit(emb)
        neighbors = nn.radius_neighbors(emb)[1]
        idx_dups = ((i, row) for i, row in enumerate(neighbors) if len(row) > 1)
        return {frozenset(ents[idx] for idx in row) for i, row in idx_dups}

    def opt(tol, info):
        s0 = time.perf_counter()
        r = len(set().union(*get_dups(tol))) / len(emb) - 0.1
        steps.append(time.perf_counter() - s0)
        print("    host step %d: tol %.6f, %.1f s" % (len(steps), tol, steps[-1]), flush=True)
        if time.perf_counter() - t0 > budget:
            raise Budget()
        return r

    # spatial.distance_matrix(emb, emb) loops over rows in numpy (minutes at this size): its time is taken on a 256-row
    # slice and scaled; the bracket's end comes from the same max computed in float64 through the Gram matrix
    s0 = time.perf_counter()
    spatial.distance_matrix(emb[:256], emb)
    t_dm = (time.perf_counter() - s0) * len(emb) / 256
    e64 = emb.astype(np.float64)
    sq = (e64 ** 2).sum(1)
    max_distance = float(np.sqrt(max(0.0, (sq[:, None] + sq[None, :] - 2.0 * e64 @ e64.T).max())))
    print("    host distance_matrix %.1f s (scaled from 256 rows)" % t_dm, flush=True)
    t0 = time.perf_counter()
    try:
        optimize.bisect(opt, 0.0, max_distance, xtol=1e-3, maxiter=50, args=({"Nfeval": 0},))
        note = "%d radius self-joins measured" % len(steps)
    except Budget:
        note = "radius self-joins extrapolated from %d measured" % len(steps)
    total = t_dm + np.mean(steps) * (len(evals) + 1)  # the bisection's steps, then the final get_dups
    print("    reference on the HOST CPU (%d cores): %.1f s (%s; distance_matrix %.1f s, %.1f s per radius self-join)"
          % (os.cpu_count(), total, note, t_dm, np.mean(steps)), flush=True)


def case_d(iters=3):
    rng = np.random.default_rng(4)
    E, b, top = 1_000_000, 1024, 10
    eng = KGEEngine("ComplEx", 200, 1, E, 1)
    eng.init_glorot_uniform(5)
    q = torch.as_tensor(rng.integers(0, E, b).astype(np.int32)).cuda()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for metric in ("euclidean", "manhattan"):
        ms = np.median(measure.per_call_ms(lambda: eng.knn(eng.ent, q, top, metric), iters, 2, before=flush.zero_))
        print("(d) kge_knn E=%d ld=400 b=%d top=%d %-9s %.2f ms (%.1f G distances/s)"
              % (E, b, top, metric, ms, b * E / ms / 1e6))
    eng.close()


if __name__ == "__main__":
    print(measure.card(), flush=True)
    which = sys.argv[1:] or ["a", "b", "c", "d"]
    for c in which:
        {"a": case_a, "b": case_b, "c": case_c, "d": case_d}[c]()
        torch.cuda.empty_cache()
