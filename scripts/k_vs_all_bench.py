#!/usr/bin/env python
"""KvsAll training benchmark (development aid): times one KvsAll step of one side (kge_k_vs_all_step,
csrc/kge_train_1vsall.cu) on the FB15k-237 shape -- 14,541 entities, 237 relations, ComplEx k = 200, random tables --
for side o and side s at B = 256, 1,000 and 4,096 queries with 1 to 20 random labels each.  In the same run it times
kge_one_vs_all_step of the same side at the same B, and the baseline a user writes in torch on the same GPU: the query
vectors, one fp32 matrix product [B, K] x [K, n_ent] with TF32 off, dense multi-hot targets, clip, the same loss,
autograd.  The script checks that the baseline's loss agrees with the kernels'.

Reported per (side, B): the step time (CUDA events around the library call, median of --iters after warm-up), the
achieved fp32 rate counted from the shapes (flops() below: 4 contractions of 2 B n_ent ld operations) and its share of
the H100 SXM's 67 TFLOP/s fp32 data-sheet peak, the 1vsAll step time and the ratio of the two, and the torch time.
Prints the GPU, its power limit and max SM clock first: every number depends on them.

    python scripts/k_vs_all_bench.py [--iters N] [--out FILE.json]
    python scripts/k_vs_all_bench.py --profile DIR   # torch.profiler kernel table of both steps at B = 1,000, side o
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import measure  # noqa: E402

E, R, K_USER = 14541, 237, 200  # FB15k-237, ComplEx k = 200
FP32_PEAK = 67e12  # H100 SXM data sheet, dense fp32, 700 W
SMOOTHING = 0.1


def flops(B, ld):
    """Operations of one side: dQ and dX each form the logits and accumulate a gradient (4 contractions), an FMA
    counted as 2."""
    return 4 * 2 * B * E * ld


def torch_step(ent, rel, t, side, y):
    """The torch baseline: dense [n_ent, 2k] tables with requires_grad, one side, reduction sum, dense targets y."""
    h = ent.shape[1] // 2
    e_s, e_p, e_o = ent[t[:, 0]], rel[t[:, 1]], ent[t[:, 2]]
    sr, si, pr, pi, orr, oi = e_s[:, :h], e_s[:, h:], e_p[:, :h], e_p[:, h:], e_o[:, :h], e_o[:, h:]
    if side == "o":
        q = torch.cat([sr * pr - si * pi, si * pr + sr * pi], 1)
    else:
        q = torch.cat([pr * orr + pi * oi, pr * oi - pi * orr], 1)
    lc = torch.clamp(q @ ent.T, -75.0, 75.0)
    loss = (torch.nn.functional.softplus(lc) - y * lc).sum()
    ent.grad = rel.grad = None
    loss.backward()
    return loss


def inputs(B, side, rng):
    """Random queries [B, 3] with 1-20 sorted distinct labels each; the answer column holds the first label."""
    labels = [np.unique(rng.integers(0, E, int(rng.integers(1, 21)))) for _ in range(B)]
    off = np.concatenate([[0], np.cumsum([len(x) for x in labels])]).astype(np.int64)
    ids = np.concatenate(labels).astype(np.int32)
    keep, p, first = rng.integers(0, E, B), rng.integers(0, R, B), ids[off[:-1]]
    q = np.stack([keep, p, first] if side == "o" else [first, p, keep], 1).astype(np.int32)
    return q, off, ids


def setup(B, side):
    from ampligraph_b200.engine import KGEEngine
    rng = np.random.default_rng(0)
    K = 2 * K_USER
    ent = rng.uniform(-0.1, 0.1, (E, K)).astype(np.float32)
    rel = rng.uniform(-0.1, 0.1, (R, K)).astype(np.float32)
    q, off, ids = inputs(B, side, rng)
    dev = lambda a: torch.as_tensor(a).cuda()
    kva = KGEEngine("ComplEx", K_USER, 1, E, R, loss="nll", optimizer="sgd")
    ova = KGEEngine("ComplEx", K_USER, 1, E, R, loss="multiclass_nll", optimizer="sgd")
    for eng in (kva, ova):
        eng.set_embeddings(ent, rel)
    tq, toff, tids = dev(q), dev(off), dev(ids)
    kva_step = lambda: kva.k_vs_all_backward(tq, side, toff, tids, SMOOTHING)
    ova_step = lambda: ova.one_vs_all_backward(tq, side)
    return ent, rel, q, off, ids, kva, ova, kva_step, ova_step


def run(B, side, iters):
    ent, rel, q, off, ids, kva, ova, kva_step, ova_step = setup(B, side)
    ms = float(np.median(measure.per_call_ms(kva_step, iters, 3)))
    ms_ova = float(np.median(measure.per_call_ms(ova_step, iters, 3)))
    # agreement with the baseline on one step from zeroed accumulators
    kva.loss_acc.zero_()
    kva_step()
    got_loss = float(kva.loss_acc[0])
    te = torch.as_tensor(ent).cuda().requires_grad_(True)
    tr = torch.as_tensor(rel).cuda().requires_grad_(True)
    tl = torch.as_tensor(q).long().cuda()
    y = torch.zeros((B, E), dtype=torch.float32, device="cuda")
    y[torch.repeat_interleave(torch.arange(B), torch.as_tensor(np.diff(off))).cuda(), torch.as_tensor(ids).long().cuda()] = 1.0
    y = (1.0 - SMOOTHING) * y + SMOOTHING / E
    base_loss = float(torch_step(te, tr, tl, side, y).detach())
    ms_torch = float(np.median(measure.per_call_ms(lambda: torch_step(te, tr, tl, side, y), iters, 3)))
    ld = kva.ld
    kva.close()
    ova.close()
    fl = flops(B, ld)
    res = {"side": side, "B": B, "ms": ms, "tflops": fl / ms * 1e-9, "share_of_fp32_peak": fl / ms * 1e3 / FP32_PEAK,
           "one_vs_all_ms": ms_ova, "ratio_to_one_vs_all": ms / ms_ova, "torch_ms": ms_torch, "loss": got_loss,
           "torch_loss": base_loss, "loss_rel_diff": abs(got_loss - base_loss) / abs(base_loss)}
    print("FB15k-237 ComplEx k=200 side %s B=%-5d  kge_k_vs_all_step %8.3f ms (%5.2f TFLOP/s fp32, %4.1f%% of 67)  "
          "kge_one_vs_all_step %8.3f ms (ratio %.2f)  torch fp32 (TF32 off) %8.3f ms  loss rel diff %.1e"
          % (side, B, ms, res["tflops"], 100 * res["share_of_fp32_peak"], ms_ova, res["ratio_to_one_vs_all"], ms_torch,
             res["loss_rel_diff"]), flush=True)
    return res


def profile(out_dir, B=1000, side="o"):
    """Kernel times of both steps at one shape under torch.profiler (a run of its own: tracing slows the host)."""
    from torch.profiler import ProfilerActivity
    from torch.profiler import profile as prof
    *_, kva, ova, kva_step, ova_step = setup(B, side)
    for fn in (kva_step, ova_step):
        fn()
    torch.cuda.synchronize()
    os.makedirs(out_dir, exist_ok=True)
    for name, fn in (("k_vs_all", kva_step), ("one_vs_all", ova_step)):
        with prof(activities=[ProfilerActivity.CUDA]) as p:
            for _ in range(10):
                fn()
            torch.cuda.synchronize()
        table = p.key_averages().table(sort_by="cuda_time_total", row_limit=12)
        print("== %s, side %s, B = %d, 10 steps ==\n%s" % (name, side, B, table), flush=True)
        with open(os.path.join(out_dir, "%s_kernels.txt" % name), "w") as f:
            f.write(table)
    kva.close()
    ova.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", default=None, metavar="DIR")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("k_vs_all_bench.py needs a GPU: times are measured on the device, never estimated")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    info = measure.card()
    print(info, flush=True)
    if args.profile:
        profile(args.profile)
        return
    results = {"gpu": info, "runs": [run(B, side, args.iters) for side in ("o", "s") for B in (256, 1000, 4096)]}
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
