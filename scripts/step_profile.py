#!/usr/bin/env python
"""Per-kernel device time of bench.py's training step (development aid): torch.profiler over N cfg2 train_steps
(the headline workload: same tables, triples and batches as bench.py), L2 flushed between steps, one line per kernel
with its mean time per step.  KGE_B200_LIB selects a variant library, e.g. one built by
scripts/build_define_variant.sh.  Usage: python scripts/step_profile.py [steps]"""
import os
import sys

import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from ampligraph_b200.engine import KGEEngine  # noqa: E402


def main(steps):
    c = bench.WORKLOADS["cfg2"]
    rng = np.random.default_rng(0)
    K = bench.internal_k(c)
    B = c["batch"]
    eng = KGEEngine(c["model"], c["k"], c["eta"], c["n_ent"], c["n_rel"], loss=c["loss"], loss_params=c["loss_params"],
                    optimizer=c["optimizer"], optimizer_params={"learning_rate": c["lr"]})
    eng.set_embeddings(bench.glorot(c["n_ent"], K, rng), bench.glorot(c["n_rel"], K, rng))
    data_np = bench.synthetic_kg(c["n_ent"], c["n_rel"], c["n_triples"])
    eng.set_hot_entities(triples=data_np)
    nb = len(data_np) // B
    data = torch.as_tensor(data_np).cuda()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for i in range(10):
        eng.train_step(data[(i % nb) * B:(i % nb + 1) * B], None, seed=1234, step=i)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(steps):
            flush.fill_(i & 0xff)
            eng.train_step(data[(i % nb) * B:(i % nb + 1) * B], None, seed=1234, step=10 + i)
        torch.cuda.synchronize()
    lib = os.path.basename(os.environ.get("KGE_B200_LIB", "libkge_b200.so"))
    for ev in sorted(prof.key_averages(), key=lambda e: -e.device_time_total):
        if "kge_" in ev.key:
            print("%-28s %9.1f us/step  %4d calls  %s" % (lib, ev.device_time_total / steps, ev.count, ev.key[:90]))
    print("%-28s loss %.9e" % (lib, eng.read_loss()))
    eng.close()


if __name__ == "__main__":
    main(int(sys.argv[1]) if len(sys.argv) > 1 else 50)
