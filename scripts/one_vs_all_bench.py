#!/usr/bin/env python
"""1vsAll training benchmark (development aid): times one 1vsAll step (kge_one_vs_all_step, csrc/kge_train_1vsall.cu;
both sides) on the FB15k-237 shape -- 14,541 entities, 237 relations, ComplEx k = 200 -- at B = 256, 1,000 and 4,096
positives, against the baseline a user writes in torch on the same GPU: the query vectors, one fp32 matrix product
[B, K] x [K, n_ent] per side with TF32 off, clip, logsumexp, autograd.  Both compute the same loss and gradients; the
script checks that they agree.

Reported per B: the step time (CUDA events around the library call, median of --iters after warm-up), the achieved fp32
rate counted from the shapes (flops() below: 5 contractions of 2 B n_ent ld operations per side) and its share of the
H100 SXM's 67 TFLOP/s fp32 data-sheet peak, and the same time for the torch baseline.  Prints the GPU and its power
limit first: every number depends on both.

    python scripts/one_vs_all_bench.py [--iters N] [--out FILE.json]
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


def flops(B, ld, sides=2):
    """Operations of the five contractions per side (stats, dQ logits + Gq, dX logits + Gx), an FMA counted as 2."""
    return sides * 5 * 2 * B * E * ld


def torch_step(ent, rel, t):
    """The torch baseline: dense [n_ent, 2k] tables with requires_grad, both sides, reduction sum."""
    h = ent.shape[1] // 2
    e_s, e_p, e_o = ent[t[:, 0]], rel[t[:, 1]], ent[t[:, 2]]
    sr, si, pr, pi, orr, oi = e_s[:, :h], e_s[:, h:], e_p[:, :h], e_p[:, h:], e_o[:, :h], e_o[:, h:]
    q_o = torch.cat([sr * pr - si * pi, si * pr + sr * pi], 1)
    q_s = torch.cat([pr * orr + pi * oi, pr * oi - pi * orr], 1)
    loss = 0.0
    for q, col in ((q_s, 0), (q_o, 2)):
        lc = torch.clamp(q @ ent.T, -75.0, 75.0)
        loss = loss + (torch.logsumexp(lc, 1) - lc.gather(1, t[:, col:col + 1])[:, 0]).sum()
    ent.grad = rel.grad = None
    loss.backward()
    return loss


def run(B, iters):
    from ampligraph_b200.engine import KGEEngine
    rng = np.random.default_rng(0)
    K = 2 * K_USER
    ent = rng.uniform(-0.1, 0.1, (E, K)).astype(np.float32)
    rel = rng.uniform(-0.1, 0.1, (R, K)).astype(np.float32)
    X = np.stack([rng.integers(0, E, B), rng.integers(0, R, B), rng.integers(0, E, B)], 1).astype(np.int32)
    t = torch.as_tensor(X).cuda()
    eng = KGEEngine("ComplEx", K_USER, 1, E, R, loss="multiclass_nll", optimizer="sgd")
    eng.set_embeddings(ent, rel)

    def step():
        eng.one_vs_all_backward(t, "s,o")
    ms = float(np.median(measure.per_call_ms(step, iters, 3)))
    # agreement with the baseline on one step from zeroed accumulators
    eng.g_ent.zero_()
    eng.g_rel.zero_()
    eng.loss_acc.zero_()
    step()
    got_loss = float(eng.loss_acc[0])
    te = torch.as_tensor(ent).cuda().requires_grad_(True)
    tr = torch.as_tensor(rel).cuda().requires_grad_(True)
    tl = torch.as_tensor(X).long().cuda()
    base_loss = float(torch_step(te, tr, tl).detach())
    ms_torch = float(np.median(measure.per_call_ms(lambda: torch_step(te, tr, tl), iters, 3)))
    ld = eng.ld
    eng.close()
    fl = flops(B, ld)
    res = {"B": B, "ms": ms, "tflops": fl / ms * 1e-9, "share_of_fp32_peak": fl / ms * 1e3 / FP32_PEAK,
           "torch_ms": ms_torch, "speedup_vs_torch": ms_torch / ms, "loss": got_loss, "torch_loss": base_loss,
           "loss_rel_diff": abs(got_loss - base_loss) / abs(base_loss)}
    print("FB15k-237 ComplEx k=200 B=%-5d  kge_one_vs_all_step %8.3f ms (%5.2f TFLOP/s fp32, %4.1f%% of 67)  "
          "torch fp32 (TF32 off) %8.3f ms (%.2fx)  loss rel diff %.1e"
          % (B, ms, res["tflops"], 100 * res["share_of_fp32_peak"], ms_torch, res["speedup_vs_torch"], res["loss_rel_diff"]),
          flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("one_vs_all_bench.py needs a GPU: times are measured on the device, never estimated")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    info = measure.card()
    print(info, flush=True)
    results = {"gpu": info, "runs": [run(B, args.iters) for B in (256, 1000, 4096)]}
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
