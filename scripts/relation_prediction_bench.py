#!/usr/bin/env python
"""Relation-prediction term benchmark (development aid): times the auxiliary 1vsAll relation step
(kge_one_vs_all_relation_step, csrc/kge_train_1vsall.cu) against the 1vsAll entity step it is added to
(kge_one_vs_all_step, sides "s,o") on the FB15k-237 shape -- 14,541 entities, 237 relations, ComplEx k = 200 -- at
B = 256, 1,000 and 4,096 positives, and against the baseline a user writes in torch: Qp = d f / dp, one fp32 matrix
product [B, K] x [K, n_rel] with TF32 off, clip, logsumexp, autograd.  Both compute the same loss and relation
gradient; the script checks that they agree.

Reported per B: both step times (CUDA events around the library call, median of --iters after warm-up), the relation
step's share of the entity step, its fp32 rate counted from the shapes (5 contractions of 2 B n_rel ld operations), the
torch baseline's time, and a torch.profiler per-kernel breakdown of the relation step (a run of its own).

With --parent-lib (a library built from the parent commit by scripts/build_variant.sh), the entity step is also timed
in worker processes that alternate the parent library and this tree's (KGE_B200_LIB), and each worker's 1vsAll ("s,o"),
relation-step and KvsAll (both sides) outputs on batches whose positives share no subject, object or relation -- so
every red.global.add target gets one add per kernel and the gradient tables are deterministic -- are compared bit for
bit: the gradient tables and losses under both reductions, and the row stamps of the looked-up-rows optimizer rule.
Prints the GPU and its power limit first: every number depends on both.

    python scripts/relation_prediction_bench.py [--iters N] [--parent-lib PATH] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import measure  # noqa: E402

E, R, K_USER = 14541, 237, 200  # FB15k-237, ComplEx k = 200
BATCHES = (256, 1000, 4096)


def tables(n_ent, n_rel, seed=0):
    rng = np.random.default_rng(seed)
    K = 2 * K_USER
    return (rng.uniform(-0.1, 0.1, (n_ent, K)).astype(np.float32), rng.uniform(-0.1, 0.1, (n_rel, K)).astype(np.float32),
            rng)


def engine(ent, rel):
    from ampligraph_b200.engine import KGEEngine
    eng = KGEEngine("ComplEx", K_USER, 1, ent.shape[0], rel.shape[0], loss="multiclass_nll", optimizer="sgd")
    eng.set_embeddings(ent, rel)
    return eng


def torch_relation_term(ent, rel, t):
    """The torch baseline of the term: Qp(s, o) @ rel.T, clip, logsumexp - l_p, reduction sum, autograd."""
    h = ent.shape[1] // 2
    e_s, e_o = ent[t[:, 0]], ent[t[:, 2]]
    sr, si, orr, oi = e_s[:, :h], e_s[:, h:], e_o[:, :h], e_o[:, h:]
    qp = torch.cat([sr * orr + si * oi, sr * oi - si * orr], 1)
    lc = torch.clamp(qp @ rel.T, -75.0, 75.0)
    loss = (torch.logsumexp(lc, 1) - lc.gather(1, t[:, 1:2])[:, 0]).sum()
    ent.grad = rel.grad = None
    loss.backward()
    return loss


def profile_kernels(fn, iters=10):
    """{kernel name: mean device ms per call of fn} from torch.profiler (CUDA activities only)."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        t_us = getattr(ev, "device_time_total", None)
        if t_us is None:
            t_us = ev.cuda_time_total
        if t_us > 0:
            out[ev.key] = t_us / 1e3 / iters
    return dict(sorted(out.items(), key=lambda kv: -kv[1]))


def run(B, iters):
    ent, rel, rng = tables(E, R)
    X = np.stack([rng.integers(0, E, B), rng.integers(0, R, B), rng.integers(0, E, B)], 1).astype(np.int32)
    t = torch.as_tensor(X).cuda()
    eng = engine(ent, rel)
    ms_ent = float(np.median(measure.per_call_ms(lambda: eng.one_vs_all_backward(t, "s,o"), iters, 3)))
    ms_rel = float(np.median(measure.per_call_ms(lambda: eng.one_vs_all_relation_backward(t, 1.0), iters, 3)))
    # agreement with the baseline on one relation step from zeroed accumulators
    eng.g_ent.zero_()
    eng.g_rel.zero_()
    eng.loss_acc.zero_()
    eng.one_vs_all_relation_backward(t, 1.0)
    torch.cuda.synchronize()
    got_loss = float(eng.loss_acc[0])
    g_rel = eng.g_rel.cpu().numpy()  # k = 200 = kp: the [re | im] rows carry no pad columns
    te = torch.as_tensor(ent).cuda().requires_grad_(True)
    tr = torch.as_tensor(rel).cuda().requires_grad_(True)
    tl = torch.as_tensor(X).long().cuda()
    base_loss = float(torch_relation_term(te, tr, tl).detach())
    base_g_rel = tr.grad.cpu().numpy()
    ms_torch = float(np.median(measure.per_call_ms(lambda: torch_relation_term(te, tr, tl), iters, 3)))
    kernels = profile_kernels(lambda: eng.one_vs_all_relation_backward(t, 1.0))
    ld = eng.ld
    eng.close()
    fl = 5 * 2 * B * R * ld
    res = {"B": B, "ms_entity_step": ms_ent, "ms_relation_step": ms_rel, "relation_share": ms_rel / ms_ent,
           "relation_tflops": fl / ms_rel * 1e-9, "torch_ms": ms_torch, "loss": got_loss, "torch_loss": base_loss,
           "loss_rel_diff": abs(got_loss - base_loss) / abs(base_loss),
           "g_rel_max_diff_rel": float(np.abs(g_rel - base_g_rel).max() / np.abs(base_g_rel).max()),
           "relation_step_kernels_ms": kernels}
    print("B=%-5d  one_vs_all_step(s,o) %8.3f ms  relation step %7.3f ms (%5.1f%% of it, %5.2f TFLOP/s fp32)  "
          "torch fp32 term %7.3f ms  loss rel diff %.1e  g_rel max diff %.1e"
          % (B, ms_ent, ms_rel, 100 * res["relation_share"], res["relation_tflops"], ms_torch, res["loss_rel_diff"],
             res["g_rel_max_diff_rel"]), flush=True)
    for name, ms in kernels.items():
        print("    %8.4f ms  %s" % (ms, name[:110]), flush=True)
    return res


def distinct_batch(n_ent, n_rel, B, rng):
    """B positives with pairwise distinct subjects, objects and relations."""
    return np.stack([rng.permutation(n_ent)[:B], rng.permutation(n_rel)[:B], rng.permutation(n_ent)[:B]],
                    1).astype(np.int32)


def worker(out_dir, iters):
    """Runs under KGE_B200_LIB: times the entity step at each B and saves deterministic outputs to out_dir."""
    import ctypes
    from ampligraph_b200 import _lib
    probe = ctypes.CDLL(_lib.SO_PATH)
    for name in list(_lib.PROTOTYPES):  # the parent build lacks this tree's newer entry points
        if not hasattr(probe, name):
            del _lib.PROTOTYPES[name]
    from ampligraph_b200.datasets import FilterIndex, k_vs_all_queries
    times = {}
    ent, rel, rng = tables(E, R)
    eng = engine(ent, rel)
    for B in BATCHES:
        t = torch.as_tensor(np.stack([rng.integers(0, E, B), rng.integers(0, R, B), rng.integers(0, E, B)],
                                     1).astype(np.int32)).cuda()
        times[B] = float(np.median(measure.per_call_ms(lambda: eng.one_vs_all_backward(t, "s,o"), iters, 3)))
    eng.close()
    outs = {}

    def save(key, eng):
        torch.cuda.synchronize()
        outs[key + "_g_ent"], outs[key + "_g_rel"] = eng.g_ent.cpu().numpy(), eng.g_rel.cpu().numpy()
        outs[key + "_loss"] = eng.loss_acc.cpu().numpy()
        if eng.lazy:
            outs[key + "_stamps_ent"], outs[key + "_stamps_rel"] = (eng.stamps[tb].cpu().numpy() for tb in ("ent", "rel"))

    from ampligraph_b200.engine import KGEEngine
    for n_rel, B in ((R, R), (4096, 4096)):  # FB15k-237's relations, and a wide relation table for B = 4,096
        ent, rel, rng = tables(E, n_rel, seed=n_rel)
        X = distinct_batch(E, n_rel, B, rng)
        # KvsAll: each positive is one query of each side, with a second label: (s, p, o + 1) and (s + 1, p, o)
        X2 = np.concatenate([X, X.copy(), X.copy()])
        X2[B:2 * B, 2] = (X[:, 2] + 1) % E
        X2[2 * B:, 0] = (X[:, 0] + 1) % E
        findex = FilterIndex(X2, E)
        kva = {side: [torch.as_tensor(a).cuda() for a in k_vs_all_queries(findex, X, side)] for side in ("o", "s")}
        t = torch.as_tensor(X).cuda()
        steps = {"ova": ("multiclass_nll", lambda eng: eng.one_vs_all_backward(t, "s,o", step=5)),
                 "ovr": ("multiclass_nll", lambda eng: eng.one_vs_all_relation_backward(t, 1.0, step=5)),
                 "kva": ("nll", lambda eng: [eng.k_vs_all_backward(q, side, off, ids, 0.1, step=5)
                                             for side, (q, off, ids) in kva.items()])}
        # every step under both reductions with SGD, and under sum with Adam's looked-up-rows rule on both tables
        for name, (loss, fn) in steps.items():
            for red, lazy in (("sum", None), ("mean", None), ("sum", (True, True))):
                eng = KGEEngine("ComplEx", K_USER, 1, E, n_rel, loss=loss, loss_params={"reduction": red},
                                optimizer="adam" if lazy else "sgd", lazy_tables=lazy)
                eng.set_embeddings(ent, rel)
                fn(eng)
                save("%s_%d_%s%s" % (name, B, red, "_lazy" if lazy else ""), eng)
                eng.close()
    np.savez(os.path.join(out_dir, "outputs.npz"), **outs)
    print(json.dumps({str(b): ms for b, ms in times.items()}), flush=True)


def ab(parent_lib, iters, rounds=2):
    """Alternates parent and new libraries in worker processes; returns the entity-step times and the comparison."""
    new_lib = os.path.join(ROOT, "ampligraph_b200", "libkge_b200.so")
    times = {"parent": [], "new": []}
    outputs = {}
    with tempfile.TemporaryDirectory() as tmp:
        for r in range(rounds):
            for name, lib in (("parent", parent_lib), ("new", new_lib)):
                d = os.path.join(tmp, "%s_%d" % (name, r))
                os.makedirs(d)
                env = dict(os.environ, KGE_B200_LIB=lib)
                out = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", d, "--iters", str(iters)],
                                     env=env, stdout=subprocess.PIPE, text=True, check=True).stdout
                times[name].append({int(k): v for k, v in json.loads(out.strip().splitlines()[-1]).items()})
                outputs.setdefault(name, dict(np.load(os.path.join(d, "outputs.npz"))))
    p, n = outputs["parent"], outputs["new"]
    cmp = {}
    for key in sorted(p):
        if key.endswith("_loss"):
            cmp[key] = float(abs(p[key][0] - n[key][0]) / abs(p[key][0]))
        else:
            cmp[key] = bool(np.array_equal(p[key].view(np.uint32), n[key].view(np.uint32)))
    print("entity step (kge_one_vs_all_step s,o) parent vs new, ms per round:", flush=True)
    for B in BATCHES:
        print("    B=%-5d parent %s  new %s" % (B, ["%.3f" % x[B] for x in times["parent"]],
                                                 ["%.3f" % x[B] for x in times["new"]]), flush=True)
    bits = all(v for k, v in cmp.items() if not k.endswith("_loss"))
    print("1vsAll / relation / KvsAll gradient tables and stamps bit-identical to the parent build: %s; largest loss rel "
          "diff %.1e"
          % (bits, max(v for k, v in cmp.items() if k.endswith("_loss"))), flush=True)
    for k, v in cmp.items():
        if not k.endswith("_loss") and not v:
            print("    differs:", k, flush=True)
    return {"times": {k: [{str(b): x for b, x in r.items()} for r in v] for k, v in times.items()}, "bits": bits,
            "compare": cmp}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("relation_prediction_bench.py needs a GPU: times are measured on the device, never estimated")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    if args.worker:
        return worker(args.worker, args.iters)
    info = measure.card()
    print(info, flush=True)
    results = {"gpu": info, "runs": [run(B, args.iters) for B in BATCHES]}
    if args.parent_lib:
        results["ab"] = ab(args.parent_lib, args.iters)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
