"""Float64 oracle of KvsAll training (kge_k_vs_all_step, DESIGN.md 3.13): the multi-label NLL of every query against
every entity with dense targets, the gradients of both tables from torch autograd, and plain-Python restatements of
the query grouping and of the epoch's batch schedule that fit(k_vs_all=...) uses.  The all-entity scores are
oracle.ref_step.corruption_scores (the reference's broadcast form) for small cases, or
one_vs_all_oracle.query_vectors(...) @ E.T (matmul=True) where the broadcast would not fit.  Test infrastructure only."""
import numpy as np
import torch

from oracle import ref_step
from one_vs_all_oracle import query_vectors


def group(triples, side):
    """Dict-loop restatement of datasets.k_vs_all_queries: -> (keys, labels) with keys the distinct (s, p) (side 'o')
    or (p, o) (side 's') in order of first appearance and labels[i] the sorted distinct answers of keys[i]."""
    labels = {}
    for s, p, o in np.asarray(triples).tolist():
        key, ans = ((s, p), o) if side == "o" else ((p, o), s)
        labels.setdefault(key, set()).add(ans)
    return list(labels), [sorted(v) for v in labels.values()]


def query_rows(keys, labels, side):
    """[n, 3] int32 query rows of `group`'s keys, the answer column holding the first label."""
    return np.array([(k[0], k[1], lab[0]) if side == "o" else (lab[0], k[0], k[1]) for k, lab in zip(keys, labels)],
                    dtype=np.int32).reshape(-1, 3)


def steps(n_o, n_s, batch_size):
    """Restatement of datasets.k_vs_all_steps: ((o_lo, o_hi), (s_lo, s_hi)) per step of one epoch."""
    if n_o == 0 or n_s == 0:
        out, lo, n = [], 0, n_o + n_s
        while lo < n:
            hi = min(lo + batch_size, n)
            out.append(((lo, hi), (0, 0)) if n_o else ((0, 0), (lo, hi)))
            lo = hi
        return out
    S = (n_o + n_s + batch_size - 1) // batch_size
    return [((i * n_o // S, (i + 1) * n_o // S), (i * n_s // S, (i + 1) * n_s // S)) for i in range(S)]


def targets(labels, n_ent, eps, device="cpu"):
    """Dense [b, n_ent] float64 targets (1 - eps) y + eps / n_ent."""
    y = torch.zeros((len(labels), n_ent), dtype=torch.float64, device=device)
    for i, lab in enumerate(labels):
        y[i, list(lab)] = 1.0
    return (1.0 - eps) * y + eps / n_ent


def side_loss(logits, y, reduction):
    """Per-query loss over all-entity logits [b, n_ent] (clipped like loss_functions.py:32-35; torch.clamp passes the
    gradient on [-75, 75] only): w * sum_e softplus(l) - y' l, w = 1 (sum) or 1 / n_ent (mean)."""
    lc = torch.clamp(logits, ref_step.CLIP_LO, ref_step.CLIP_HI)
    per = (torch.logaddexp(torch.zeros_like(lc), lc) - y * lc).sum(1)
    return per / lc.shape[1] if reduction == "mean" else per


def loss_and_grads(model, ent, rel, queries, labels, side, reduction="sum", eps=0.0, device="cpu", matmul=False,
                   dtype=torch.float64):
    """(loss, g_ent, g_rel) of one KvsAll step of one side on dense tables ent [n_ent, K], rel [n_rel, K]; queries [b, 3],
    labels a list of b label lists.  In float64; dtype float32 evaluates the same graph in fp32."""
    E = torch.as_tensor(np.asarray(ent), dtype=dtype, device=device).clone().requires_grad_(True)
    R = torch.as_tensor(np.asarray(rel), dtype=dtype, device=device).clone().requires_grad_(True)
    total = _side_total(model, E, R, queries, labels, side, reduction, eps, device, matmul)
    total.backward()
    return float(total.detach()), E.grad.cpu().numpy(), R.grad.cpu().numpy()


def _side_total(model, E, R, queries, labels, side, reduction, eps, device, matmul):
    t = torch.as_tensor(np.asarray(queries), dtype=torch.long, device=device).reshape(-1, 3)
    e_s, e_p, e_o = E[t[:, 0]], R[t[:, 1]], E[t[:, 2]]
    if matmul:
        logits = query_vectors(model, side, e_s, e_p, e_o) @ E.T
    else:
        logits = ref_step.corruption_scores(model, side, e_s, e_p, e_o, E)
    return side_loss(logits, targets(labels, E.shape[0], eps, device).to(E.dtype), reduction).sum()


def fit_sgd(model, ent, rel, triples, sides, batch_size, epochs, lr, reduction="sum", eps=0.0):
    """The tables after fit(k_vs_all=sides, ...) with plain SGD (no regulariser), in float64: the same grouping and
    step schedule, one gradient over both sides' slices per step, then x -= lr * g on both tables."""
    E = torch.as_tensor(np.asarray(ent), dtype=torch.float64).clone()
    R = torch.as_tensor(np.asarray(rel), dtype=torch.float64).clone()
    grouped = {side: group(triples, side) for side in sides.split(",")}
    rows = {side: (query_rows(k, lab, side), lab) for side, (k, lab) in grouped.items()}
    count = lambda side: len(rows[side][1]) if side in rows else 0
    schedule = steps(count("o"), count("s"), batch_size)
    for _ in range(epochs):
        for ranges in schedule:
            Eg, Rg = E.clone().requires_grad_(True), R.clone().requires_grad_(True)
            total = torch.zeros((), dtype=torch.float64)
            for side, (lo, hi) in zip(("o", "s"), ranges):
                if hi > lo:
                    q, lab = rows[side]
                    total = total + _side_total(model, Eg, Rg, q[lo:hi], lab[lo:hi], side, reduction, eps, "cpu", True)
            total.backward()
            E, R = E - lr * Eg.grad, R - lr * Rg.grad
    return E.numpy(), R.numpy()
