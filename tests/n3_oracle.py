"""n3_oracle.py -- TEST INFRASTRUCTURE: the N3 regulariser of a step's positives in float64 under torch autograd.

L_N3 = lambda_ent * sum_b sum_d (|s_bd|^3 + |o_bd|^3) + lambda_rel * sum_b sum_d |p_bd|^3 over the positives
(s_b, p_b, o_b), written per occurrence (a row used twice is gathered twice), on dense tables [rows, K]: |z_d| is |x[d]|
for TransE and DistMult and the modulus of (x[d], x[k + d]) for ComplEx, HolE and RotatE (DESIGN.md 3.15).  The modulus
goes through exact_oracle._Modulus, whose gradient is 0 at 0 (m^3 has gradient 0 there).

bound() gives the per-element error bound of kge_n3_step's fp32 arithmetic (derived in its docstring).
"""
import math

import numpy as np
import torch

from exact_oracle import FP32_EPS, FP32_TINY, _Modulus

TWO_HALVES = ("ComplEx", "HolE", "RotatE")


def cubes(model, x):
    """|z_d|^3 per row of a dense [n, K] tensor -> [n, K / halves]."""
    if model in TWO_HALVES:
        h = x.shape[1] // 2
        m = _Modulus.apply(x[:, :h], x[:, h:])
    else:
        m = x.abs()
    return m * m * m


def loss_and_grads(model, ent, rel, triples, lam_ent, lam_rel, device="cpu", dtype=torch.float64):
    """(L_N3, g_ent, g_rel) of the positives `triples` [B, 3] on dense tables ent [n_ent, K], rel [n_rel, K], per
    occurrence.  The lambdas are taken as fp32 values (what the kernel receives)."""
    lam_ent, lam_rel = float(np.float32(lam_ent)), float(np.float32(lam_rel))
    E = torch.as_tensor(np.asarray(ent), dtype=dtype, device=device).clone().requires_grad_(True)
    R = torch.as_tensor(np.asarray(rel), dtype=dtype, device=device).clone().requires_grad_(True)
    t = torch.as_tensor(np.asarray(triples), dtype=torch.long, device=device).reshape(-1, 3)
    total = torch.zeros((), dtype=dtype, device=device)
    if lam_ent > 0:
        total = total + lam_ent * (cubes(model, E[t[:, 0]]).sum() + cubes(model, E[t[:, 2]]).sum())
    if lam_rel > 0:
        total = total + lam_rel * cubes(model, R[t[:, 1]]).sum()
    total.backward()
    zero = lambda T: torch.zeros_like(T).cpu().numpy()
    return (float(total.detach()), E.grad.cpu().numpy() if E.grad is not None else zero(E),
            R.grad.cpu().numpy() if R.grad is not None else zero(R))


def counts(triples, n_ent, n_rel):
    """c_row: occurrences of each entity row as s or o, and of each relation row as p."""
    t = np.asarray(triples, np.int64).reshape(-1, 3)
    return (np.bincount(np.concatenate([t[:, 0], t[:, 2]]), minlength=n_ent),
            np.bincount(t[:, 1], minlength=n_rel))


def bound(model, ent, rel, triples, lam_ent, lam_rel, k):
    """Per-element bounds of kge_n3_step against loss_and_grads, on dense tables -> (loss bound, g_ent bound [n_ent, K],
    g_rel bound [n_rel, K]) in float64.

    The kernel forms, once per row with c occurrences, coef = fl(fl(3 lambda) c), m = fl(sqrt(fl(fl(re^2) + fl(im^2))))
    (one half: m = |x|, exact), and adds fl(fl(coef m) z) to the gradient element.  With u = 2^-24 each rounding is a
    factor (1 + d), |d| <= u, and sqrt halves the relative error of its argument: the argument carries 2u (two positive
    terms squared, then added), so m carries 2u; coef 2u; the product two more.  The N3 term is then within 6u (two
    halves) or 4u (one half) of c 3 lambda m z, plus the second-order terms; 8u covers both.  Adding it to a gradient
    element is one more rounding, which the caller's bound of the element's other terms covers (u of the result).  The
    loss: each m^3 carries 3 * 2u + 2u = 8u (one half: 2u); a lane sums 4 ceil(kp / 128) of them in sequence and the
    warp's butterfly adds 5 levels, so the row sum carries (4 ceil(kp / 128) + 5) u of sum m^3 more; the fp64 products
    and the atomic add 2^-50 relative.  FP32_TINY terms cover results below the smallest normal."""
    lam_ent, lam_rel = float(np.float32(lam_ent)), float(np.float32(lam_rel))
    ce, cr = counts(triples, ent.shape[0], rel.shape[0])
    out = []
    for table, c, lam in ((ent, ce, lam_ent), (rel, cr, lam_rel)):
        x = np.abs(np.asarray(table, np.float64))
        if model in TWO_HALVES:
            h = x.shape[1] // 2
            m = np.sqrt(x[:, :h] ** 2 + x[:, h:] ** 2)
            m = np.concatenate([m, m], 1)
        else:
            m = x
        g = 3.0 * lam * c[:, None] * m * x
        out.append(8 * FP32_EPS * g + FP32_TINY * (c[:, None] > 0) * (1.0 + 3.0 * lam * c[:, None]))
    loss, _, _ = loss_and_grads(model, ent, rel, triples, lam_ent, lam_rel)
    chain = (8 if model in TWO_HALVES else 2) + 4 * math.ceil(k / 128) + 5 + 1
    return chain * FP32_EPS * loss + 2.0 ** -50 * loss + FP32_TINY, out[0], out[1]
