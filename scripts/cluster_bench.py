#!/usr/bin/env python
"""DBSCAN benchmark (development aid): KGEEngine.dbscan per phase and find_clusters end to end.

  (a) the cfg2-shaped entity table (14,505 x 400 rows of ComplEx k = 200 after one epoch, as in knn_bench.py (c)),
      eps = the median distance to the 5th nearest other row, min_samples = 5; find_clusters end to end with sklearn's
      DBSCAN at that eps, and sklearn's DBSCAN(eps, 5).fit_predict on the host CPU once -- a host number, labelled so;
  (b) the same rows with eps above the largest distance: every pair in radius, every union contends for one root;
  (c) 100,000 x 400 synthetic blobs (1,000 centres, 5 % uniform noise).
Each phase -- count sweep, core compaction (the one synchronisation), union sweep, flatten, border sweep, relabel -- is
timed with CUDA events after an L2 flush; medians over the iterations.  The total is compared with one count sweep
over the same rows.  Prints the GPU and its power limit, because every number depends on both."""
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import measure  # noqa: E402
from ampligraph_b200.engine import DBSCAN_BATCH, INT32_MAX, KGEEngine, dbscan_labels  # noqa: E402

PHASES = ("count", "compact", "union", "flatten", "border", "relabel")


def phases(eng, pts, eps, ms, metric, flush, iters):
    """KGEEngine.dbscan's steps one by one, each between two CUDA events -> ({phase: median ms}, labels)."""
    n, batch = pts.shape[0], DBSCAN_BATCH
    every = torch.arange(n, dtype=torch.int32, device="cuda")
    res = {p: [] for p in PHASES}
    for it in range(iters + 1):  # the first run warms up
        flush.fill_(it)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(PHASES) + 1)]
        ev[0].record()
        counts = torch.empty(n, dtype=torch.int64, device="cuda")
        for s in range(0, n, batch):
            counts[s:s + batch] = eng.radius_counts(pts, every[s:s + batch], eps, metric, n_cand=n)
        ev[1].record()
        core = counts >= ms
        core_ids = torch.nonzero(core).flatten().to(torch.int32)
        parent = every.clone()
        ev[2].record()
        for s in range(0, core_ids.numel(), batch):
            eng.radius_union(pts, core_ids[s:s + batch], eps, metric, parent, cand_ids=core_ids[s:])
        ev[3].record()
        eng.forest_flatten(parent)
        ev[4].record()
        border = torch.full((n,), INT32_MAX, dtype=torch.int32, device="cuda")
        if core_ids.numel() > 0:
            rest = torch.nonzero(~core).flatten().to(torch.int32)
            for s in range(0, rest.numel(), batch):
                q = rest[s:s + batch]
                border[q.long()] = eng.radius_min_key(pts, q, eps, metric, parent, cand_ids=core_ids)
        ev[5].record()
        labels = dbscan_labels(core, parent, border)
        ev[6].record()
        torch.cuda.synchronize()
        if it:
            for i, p in enumerate(PHASES):
                res[p].append(ev[i].elapsed_time(ev[i + 1]))
    want = eng.dbscan(pts, eps, ms, metric)[0]
    assert torch.equal(labels, want), "the restated phases disagree with KGEEngine.dbscan"
    return {p: float(np.median(v)) for p, v in res.items()}, labels, int(core.sum())


def report(tag, eng, pts, eps, ms, metric, flush, iters):
    t, labels, n_core = phases(eng, pts, eps, ms, metric, flush, iters)
    total = sum(t.values())
    lab = labels.cpu().numpy()
    print("(%s) n=%d ld=%d %s eps=%.6g min_samples=%d: %d clusters, %d core, %d noise" % (
        tag, pts.shape[0], pts.shape[1], metric, eps, ms, lab.max() + 1, n_core, int((lab == -1).sum())))
    print("    " + ", ".join("%s %.2f ms" % (p, t[p]) for p in PHASES))
    print("    total %.2f ms = %.2f x the count sweep" % (total, total / t["count"]), flush=True)
    return lab


def cfg2_model():
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
    return m, np.unique(X[:, 0])


def case_ab(iters=5):
    from sklearn.cluster import DBSCAN
    from ampligraph_b200.discovery import _points, find_clusters
    m, ents = cfg2_model()
    eng = m.engine
    pts = _points(m, eng, ents, "e")
    n = pts.shape[0]
    every = torch.arange(n, dtype=torch.int32, device="cuda")
    d5 = torch.cat([eng.knn(pts, every[s:s + 1024], 6, "euclidean")[1][:, 5] for s in range(0, n, 1024)])
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    report("a", eng, pts, float(d5.quantile(0.5)), 5, "euclidean", flush, iters)
    eps = float(d5.quantile(0.05))  # fewer core rows: many small clusters
    lab = report("a", eng, pts, eps, 5, "euclidean", flush, iters)

    find_clusters(ents, m, DBSCAN(eps=eps, min_samples=5))  # warm-up
    runs = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        got = find_clusters(ents, m, DBSCAN(eps=eps, min_samples=5))
        runs.append(time.perf_counter() - t0)
    print("    find_clusters(mode='e', DBSCAN(eps, 5)) end to end: %.1f ms (median of 3)" % (np.median(runs) * 1e3))
    emb = m.get_embeddings(ents, embedding_type="e")
    t0 = time.perf_counter()
    host = DBSCAN(eps=eps, min_samples=5).fit_predict(emb)
    host_s = time.perf_counter() - t0
    print("    sklearn DBSCAN(eps, 5).fit_predict on the HOST CPU (%d cores): %.1f s; labels equal: %s (GPU: %s)"
          % (os.cpu_count(), host_s, bool((host == got).all()), bool((lab == got).all())), flush=True)

    far = max(float(eng.knn(pts, every[s:s + 1024], 1, "euclidean", farthest=True)[1].max()) for s in range(0, n, 1024))
    report("b", eng, pts, far * 1.01, 5, "euclidean", flush, iters)


def case_c(iters=3):
    n, ld = 100_000, 400
    g = torch.Generator(device="cuda").manual_seed(9)
    centers = torch.rand((1000, ld), generator=g, device="cuda") - 0.5
    pts = centers[torch.randint(0, 1000, (n,), generator=g, device="cuda")]
    pts += 0.035 * torch.randn((n, ld), generator=g, device="cuda")
    far = torch.rand(n, generator=g, device="cuda") < 0.05
    pts[far] = torch.rand((int(far.sum()), ld), generator=g, device="cuda") - 0.5
    pts = pts.contiguous()
    eng = KGEEngine("TransE", 4, 1, 8, 1)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    report("c", eng, pts, 1.0, 10, "euclidean", flush, iters)
    eng.close()


if __name__ == "__main__":
    print(measure.card(), flush=True)
    which = sys.argv[1:] or ["ab", "c"]
    for c in which:
        {"ab": case_ab, "c": case_c}[c]()
        torch.cuda.empty_cache()
