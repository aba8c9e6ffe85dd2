#!/usr/bin/env python
"""Top-k link-prediction micro-benchmark (development aid): times kge_topk (engine.topk) against kge_corruption_scores
alone and kge_corruption_scores + torch.topk on the same queries.  torch.topk is the obvious alternative, not a parity
reference (it does not promise the tie order).  CUDA events, L2 flushed between iterations; prints the GPU and its power
limit, because every number depends on both."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import measure  # noqa: E402
from ampligraph_b200.engine import KGEEngine  # noqa: E402


def run(model, k, E, b, top, sides=("o", "s"), iters=10, R=237):
    rng = np.random.default_rng(0)
    eng = KGEEngine(model, k, 1, E, R)
    eng.init_glorot_uniform(1)
    t = torch.as_tensor(np.stack([rng.integers(0, E, b), rng.integers(0, R, b), rng.integers(0, E, b)], 1)
                        .astype(np.int32)).cuda()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    ws = eng.lib.kge_topk_workspace_bytes(eng.h, b, E, top)
    median_ms = lambda fn: float(np.median(measure.per_call_ms(fn, iters, 2, before=flush.zero_)))
    for side in sides:
        t_topk = median_ms(lambda: eng.topk(t, side, top))
        t_cs = median_ms(lambda: eng.corruption_scores(t, side))
        t_cst = median_ms(lambda: torch.topk(eng.corruption_scores(t, side), top, dim=1))
        print("%-8s k=%-4d E=%-8d b=%-5d top=%-4d side=%s  topk %9.1f us  scores %9.1f us  scores+torch.topk %9.1f us  "
              "topk/scores %.3f  workspace %.1f MB (score matrix %.1f MB)"
              % (model, k, E, b, top, side, t_topk * 1e3, t_cs * 1e3, t_cst * 1e3, t_topk / t_cs, ws / 2**20,
                 4.0 * b * E / 2**20), flush=True)
    eng.close()
    del flush
    torch.cuda.empty_cache()


def chunk_sweep():
    """kge_topk time against the candidates per chunk (KGE_B200_TOPK_CHUNK, read when the handle is created)."""
    for E, b, chunks in ((14505, 1024, (4864, 6144, 7424, 8448, 12288, 14592)), (1000000, 1024, (6144, 8448, 16384))):
        for c in chunks:
            os.environ["KGE_B200_TOPK_CHUNK"] = str(c)
            print("chunk %d (%.1f MB)" % (c, 4.0 * b * c / 2**20), end=": ", flush=True)
            run("ComplEx", 200, E, b, 10, sides=("o",), iters=3 if E > 100000 else 10)
    del os.environ["KGE_B200_TOPK_CHUNK"]


if __name__ == "__main__":
    print(measure.card(), flush=True)
    if "--chunk-sweep" in sys.argv:
        chunk_sweep()
        sys.exit(0)
    run("ComplEx", 200, 14505, 1024, 10)        # cfg2 table
    run("ComplEx", 200, 14505, 1024, 100)
    run("ComplEx", 200, 14505, 1, 10)           # a single query_topn
    run("TransE", 400, 14505, 1024, 10)
    run("RotatE", 200, 14505, 1024, 10)
    run("ComplEx", 200, 1000000, 1024, 10, sides=("o",), iters=3)
