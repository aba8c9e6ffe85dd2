"""dura_oracle.py -- TEST INFRASTRUCTURE: the DURA regulariser of a step's positives in float64 under torch autograd.

L_DURA = sum_b sum_d [ w_n (m_h + m_t) + w_p m_r (m_h + m_t) ] over the positives (h_b, r_b, t_b), written per occurrence
(a row used twice is gathered twice), on dense tables [rows, K]: m_x = x[d]^2 for DistMult and x[d]^2 + x[k + d]^2 for
ComplEx and HolE (DESIGN.md 3.16).

closed_form() restates the gradient per row (sums over each row's occurrences, the form the kernel's REDs add up), and
bound() gives the per-element error bound of kge_dura_step's fp32 arithmetic (derived in its docstring).
"""
import numpy as np
import torch

from exact_oracle import FP32_EPS, FP32_TINY

TWO_HALVES = ("ComplEx", "HolE")


def squares(model, x):
    """m_d = |z_d|^2 per row of a dense [n, K] array or tensor -> [n, K / halves]."""
    m = x * x
    if model in TWO_HALVES:
        h = x.shape[1] // 2
        m = m[:, :h] + m[:, h:]
    return m


def _halves(model, v):
    """[n, K / halves] -> [n, K]: the same value for the real and the imaginary half."""
    return np.concatenate([v, v], 1) if model in TWO_HALVES else v


def weights32(w_n, w_p):
    """The weights as the fp32 values the kernel receives."""
    return float(np.float32(w_n)), float(np.float32(w_p))


def loss_and_grads(model, ent, rel, triples, w_n, w_p, device="cpu", dtype=torch.float64):
    """(L_DURA, g_ent, g_rel) of the positives `triples` [B, 3] on dense tables ent [n_ent, K], rel [n_rel, K], per
    occurrence, by autograd."""
    w_n, w_p = weights32(w_n, w_p)
    E = torch.as_tensor(np.asarray(ent), dtype=dtype, device=device).clone().requires_grad_(True)
    R = torch.as_tensor(np.asarray(rel), dtype=dtype, device=device).clone().requires_grad_(True)
    t = torch.as_tensor(np.asarray(triples), dtype=torch.long, device=device).reshape(-1, 3)
    s = squares(model, E[t[:, 0]]) + squares(model, E[t[:, 2]])
    total = (w_n * s).sum() + (w_p * squares(model, R[t[:, 1]]) * s).sum()
    total.backward()
    zero = lambda T: torch.zeros_like(T).cpu().numpy()
    return (float(total.detach()), E.grad.cpu().numpy() if E.grad is not None else zero(E),
            R.grad.cpu().numpy() if R.grad is not None else zero(R))


def closed_form(model, ent, rel, triples, w_n, w_p):
    """(g_ent, g_rel) per row: d/dx of an entity row = 2 x sum over its occurrences as h or t of (w_n + w_p m_r); d/dr =
    2 w_p r sum over its occurrences of (m_h + m_t)."""
    w_n, w_p = weights32(w_n, w_p)
    ent, rel = np.asarray(ent, np.float64), np.asarray(rel, np.float64)
    t = np.asarray(triples, np.int64).reshape(-1, 3)
    a = w_n + w_p * squares(model, rel[t[:, 1]])                    # [B, K / halves]
    s = squares(model, ent[t[:, 0]]) + squares(model, ent[t[:, 2]])
    ca = np.zeros((ent.shape[0], a.shape[1]))
    np.add.at(ca, t[:, 0], a)
    np.add.at(ca, t[:, 2], a)
    cs = np.zeros((rel.shape[0], s.shape[1]))
    np.add.at(cs, t[:, 1], s)
    return 2.0 * _halves(model, ca) * ent, 2.0 * w_p * _halves(model, cs) * rel


def occurrences(triples, n_ent, n_rel):
    """Occurrences of each entity row as h or t, and of each relation row as r."""
    t = np.asarray(triples, np.int64).reshape(-1, 3)
    return (np.bincount(np.concatenate([t[:, 0], t[:, 2]]), minlength=n_ent),
            np.bincount(t[:, 1], minlength=n_rel))


def bound(model, ent, rel, triples, w_n, w_p):
    """Per-element bounds of kge_dura_step against loss_and_grads, on dense tables -> (loss bound, g_ent bound
    [n_ent, K], g_rel bound [n_rel, K]) in float64.

    With u = 2^-24 each fp32 rounding is a factor (1 + d), |d| <= u.  Per occurrence and component the kernel forms
    m = fl(fl(re^2) + fl(im^2)) (2u; one half: fl(re^2), u), a = fl(w_n + fl(w_p m_r)) (2u more) and s = fl(m_h + m_t)
    (3u), and adds fl(fl(2a) x) to the entity element (2a is exact: 5u) and fl(fl(2 w_p s) r) to the relation element
    (5u).  Every term of an element has the element's sign (a, s >= 0), so the REDs' sum of its n terms, in any order,
    carries at most (n - 1) u of the sum of |terms|.  6u covers the terms with their second-order parts: the bound is
    (6 + n) u sum |term|.  A lost or doubled occurrence of a row with few of them moves the element by a whole term, far
    outside it.  The loss: each term fl(s a) carries 8u; the terms are summed in fp64, n_terms 2^-53 of the loss.
    FP32_TINY terms cover results below the smallest normal."""
    w_n, w_p = weights32(w_n, w_p)
    A_ent, A_rel = closed_form(model, np.abs(ent), np.abs(rel), triples, w_n, w_p)  # sum of |terms| per element
    ce, cr = occurrences(triples, ent.shape[0], rel.shape[0])
    b_ent = (6 + ce[:, None]) * FP32_EPS * A_ent + FP32_TINY * (ce[:, None] > 0)
    b_rel = (6 + cr[:, None]) * FP32_EPS * A_rel + FP32_TINY * (cr[:, None] > 0)
    loss, _, _ = loss_and_grads(model, ent, rel, triples, w_n, w_p)
    n_terms = np.asarray(triples).reshape(-1, 3).shape[0] * squares(model, np.asarray(ent[:1])).shape[1]
    return 8 * FP32_EPS * loss + n_terms * (2.0 ** -53 * loss + FP32_TINY), b_ent, b_rel
