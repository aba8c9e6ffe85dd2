#!/usr/bin/env python
"""Fact-discovery benchmark (development aid): the per-node wedge counts and generate_candidates / discover_facts.

  (a) the cfg2-shaped graph of bench.synthetic_kg(14505, 237, 272115) (counters in shared memory) and the YAGO3-10-
      shaped graph of bench.synthetic_kg(123182, 37, 1079040) (counters in workspace slices): the CSR build
      (engine.graph_csr, torch on the device) and the kge_graph_counts kernel, each between CUDA events, medians;
  (b) on the cfg2 graph with string labels, generate_candidates for one relation and discover_facts with
      target_rel=None (237 relations, one evaluate) for every strategy, host clock around work that ends in a
      synchronising copy, on a ComplEx model trained for one epoch;
  (c) --networkx: the host statistics the reference computes (nx.triangles, nx.clustering, nx.square_clustering over
      the first 200 nodes, scaled) and its filter's dense [|A|, |B|, 3] row comparison for 40 candidate rows, scaled
      to one sampling round (400 rows) -- host numbers, single-threaded, labelled so.
Prints the GPU and its power limit, because every number depends on both; writes the JSON to --out if given."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import measure  # noqa: E402
from ampligraph_b200 import discovery  # noqa: E402
from ampligraph_b200.engine import graph_counts_csr, graph_csr  # noqa: E402

STRATEGIES = ("random_uniform", "entity_frequency", "graph_degree", "cluster_coefficient", "cluster_triangles",
              "cluster_squares")


def kernel_arm(name, t, n, iters):
    td = torch.as_tensor(t).cuda()
    csr = graph_csr(td, n)
    degree, d, offsets, nbr, order = csr
    wedges = int((d * d).sum())
    res = {"graph": name, "nodes": n, "edges": int(nbr.numel() // 2), "max_d": int(d.max()), "wedges": wedges,
           "csr_ms": float(np.median(measure.per_call_ms(lambda: graph_csr(td, n), iters, 1))),
           "kernel_ms": float(np.median(measure.per_call_ms(lambda: graph_counts_csr(offsets, nbr, order), iters, 1)))}
    res["wedges_per_s"] = 2 * wedges / (res["kernel_ms"] * 1e-3)  # pass 1 and pass 3 each walk every wedge
    print(json.dumps(res), flush=True)
    return res


def host_clock(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--networkx", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    info = measure.card()
    print(info, flush=True)
    out = {"gpu": info, "kernel": [], "discovery": []}

    t = bench.synthetic_kg(14505, 237, 272115)
    out["kernel"].append(kernel_arm("cfg2", t[:, [0, 1, 2]], 14505, args.iters))
    y = bench.synthetic_kg(123182, 37, 1079040)
    out["kernel"].append(kernel_arm("yago3-10 shaped", y, 123182, max(3, args.iters // 3)))

    X = np.stack([np.char.add("e", t[:, 0].astype(str)), np.char.add("r", t[:, 1].astype(str)),
                  np.char.add("e", t[:, 2].astype(str))], 1).astype(object)
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    model = ScoringBasedEmbeddingModel(eta=5, k=100, scoring_type="ComplEx", seed=0)
    model.compile(optimizer="adam", loss="multiclass_nll")
    model.fit(X, batch_size=10000, epochs=1, verbose=False)
    for strategy in STRATEGIES:
        discovery.generate_candidates(X, strategy, "r0", 100)  # warm-up
        gen_s, c = host_clock(lambda: discovery.generate_candidates(X, strategy, "r0", 100))
        fact_s, (facts, ranks) = host_clock(lambda: discovery.discover_facts(X, model, top_n=10, strategy=strategy,
                                                                             max_candidates=100))
        res = {"strategy": strategy, "generate_candidates_s": gen_s, "candidates": len(c),
               "discover_facts_all_relations_s": fact_s, "facts": len(facts)}
        print(json.dumps(res), flush=True)
        out["discovery"].append(res)

    if args.networkx:
        import networkx as nx
        G = nx.Graph()
        G.add_edges_from(zip(t[:, 0].tolist(), t[:, 2].tolist()))
        host = {}
        for name, fn in (("triangles", nx.triangles), ("clustering", nx.clustering)):
            t0 = time.perf_counter()
            fn(G)
            host[name + "_s"] = time.perf_counter() - t0
        nodes = list(G)[:200]
        t0 = time.perf_counter()
        nx.square_clustering(G, nodes)
        host["square_clustering_s_scaled"] = (time.perf_counter() - t0) * G.number_of_nodes() / len(nodes)
        A = X[:40].copy()
        t0 = time.perf_counter()
        (A[:, None, :] == X[None, :, :]).all(2)
        host["dense_filter_400_rows_s_scaled"] = (time.perf_counter() - t0) * 10
        host["note"] = "host CPU, single-threaded, networkx %s" % nx.__version__
        print(json.dumps(host), flush=True)
        out["networkx"] = host
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
