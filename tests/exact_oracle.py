"""exact_oracle.py -- TEST INFRASTRUCTURE: one training step in float64, and tables on which fp32 is exact.

On tables whose entries lie on a coarse dyadic grid (multiples of 2^-f with few significant bits) every score, every
dL/dscore of the margin losses and every partial sum of a gradient element is a multiple of a fixed power of two well
below 2^24 of that unit, so every fp32 operation a training kernel performs is exact in ANY order (the red.global.add
atomics and the bucket sums included).  The kernel's result must then EQUAL this oracle's, element for element.

The oracle is oracle/ref_step.py's dtype-agnostic pieces (compute_scores, per_positive_loss, corrupt) under torch
autograd in float64; ref_step.RefStep is not used (it casts to fp32).  One deliberate deviation: RotatE's gradient at an
exactly zero residual, where the reference's sqrt gradient is NaN and the kernel's rot_unit (kge_train_common.cuh)
returns 0 -- the oracle's modulus gradient is 0 there too (_Modulus).

For the losses whose dL/dscore is not exact (nll, multiclass_nll, self_adversarial) the oracle also returns a
per-element error budget: A = sum over the element's terms of |dL/dscore_j| * |d score_j / d element| (bounds), its term
count n, and A1 = sum of |d score_j / d element| (for results below fp32's smallest normal); see grad_bound.
"""
from collections import namedtuple

import numpy as np
import torch

from oracle import ref_step

TRILINEAR = ("DistMult", "ComplEx", "HolE")
FP32_EPS = 2.0 ** -24   # unit roundoff of fp32
FP32_TINY = 2.0 ** -126  # smallest normal fp32

Step = namedtuple("Step", "loss sp sn g_ent g_rel dsp dsn mag_pos mag_neg corr")


def internal_k(model, k):
    return k if model in ("TransE", "DistMult") else 2 * k


# --------------------------------------------------------------------------
# dyadic tables
# --------------------------------------------------------------------------
GRID5 = np.array([-1.0, -0.5, 0.0, 0.5, 1.0])


def grid_table(rng, rows, cols, values=GRID5):
    """float32 [rows, cols] with entries drawn from `values` (default {-1, -1/2, 0, 1/2, 1}: 2 significant bits)."""
    return rng.choice(np.asarray(values, np.float64), (rows, cols)).astype(np.float32)


def dyadic_table(rng, rows, cols, frac_bits=4, int_bits=0):
    """float32 [rows, cols] of multiples of 2^-frac_bits in (-2^int_bits, 2^int_bits): frac_bits + int_bits + 1 bits."""
    lim = 2 ** (frac_bits + int_bits)
    return (rng.integers(-lim + 1, lim, (rows, cols)) * 2.0 ** -frac_bits).astype(np.float32)


def assert_fp32_exact(x, what=""):
    """x (float64 tensor / array) is exactly representable in fp32."""
    x = torch.as_tensor(x, dtype=torch.float64)
    bad = x != x.float().double()
    assert not bool(bad.any()), "%s: %d values not exact in fp32, e.g. %r" % (what, int(bad.sum()), x[bad][:3].tolist())


# --------------------------------------------------------------------------
# scores
# --------------------------------------------------------------------------
class _Modulus(torch.autograd.Function):
    """sqrt(re^2 + im^2) whose gradient is 0 where the modulus is 0 (the reference's is NaN there; the kernel's rot_unit,
    kge_train_common.cuh, takes g * 0 * rsqrt(max(x, tiny)) = 0)."""

    @staticmethod
    def forward(ctx, re, im):
        r = torch.sqrt(re * re + im * im)
        ctx.save_for_backward(re, im, r)
        return r

    @staticmethod
    def backward(ctx, g):
        re, im, r = ctx.saved_tensors
        safe = torch.where(r > 0, r, torch.ones_like(r))
        unit = torch.where(r > 0, g / safe, torch.zeros_like(r))
        return unit * re, unit * im


def scores(model, e_s, e_p, e_o, max_rel_size=None):
    """ref_step.compute_scores, but RotatE's modulus through _Modulus."""
    if model != "RotatE":
        return ref_step.compute_scores(model, e_s, e_p, e_o, max_rel_size)
    h = e_s.shape[1] // 2
    div = ref_step.rotate_divisor(e_s.shape[1], max_rel_size if max_rel_size else 1)
    theta = e_p[:, :h]
    p_re, p_im = torch.cos(theta / div), torch.sin(theta / div)
    re = e_s[:, :h] * p_re - e_s[:, h:] * p_im - e_o[:, :h]
    im = e_s[:, :h] * p_im + e_s[:, h:] * p_re - e_o[:, h:]
    return -torch.sum(_Modulus.apply(re, im), dim=1)


def abs_scores(model, e_s, e_p, e_o):
    """On |tables|: per triple, a function whose gradient w.r.t. each element bounds |d score / d element| (every
    product term counted positive).  TransE: 1 per element of s, p and o (|d score / d x| <= 1)."""
    if model == "TransE":
        return (e_s + e_p + e_o).sum(1)
    if model == "DistMult":
        return torch.sum(e_s * e_p * e_o, dim=1)
    h = e_s.shape[1] // 2
    s_re, s_im, p_re, p_im, o_re, o_im = e_s[:, :h], e_s[:, h:], e_p[:, :h], e_p[:, h:], e_o[:, :h], e_o[:, h:]
    # (RotatE has no bound here: its training arithmetic uses approximate sqrt / rsqrt)
    sc = torch.sum(s_re * (p_re * o_re + p_im * o_im) + s_im * (p_re * o_im + p_im * o_re), dim=1)
    return sc * (2.0 / h) if model == "HolE" else sc


# --------------------------------------------------------------------------
# loss magnitudes: per score, a bound on the terms that make up its dL/dscore
# --------------------------------------------------------------------------
def loss_magnitudes(name, sp, sn, lp, dsp, dsn):
    """float64 (mag_pos [B], mag_neg [eta, B]): |dL/dscore|, except where the loss forms dL/dscore as a difference of
    larger quantities -- multiclass_nll's dP = P/D - 1 (magnitude P/D + 1) and self_adversarial's
    dN_j = w (p_j sig_j - alpha p_j (l_j - S)) (magnitude w p_j (sig_j + alpha (|l_j| + |S|)))."""
    sp, sn = sp.detach(), sn.detach()
    mag_pos, mag_neg = dsp.detach().abs(), dsn.detach().abs()
    eta = sn.shape[0]
    w = 1.0 / eta if lp.get("reduction", "sum") == "mean" else 1.0
    if name == "multiclass_nll":
        lo, hi = ref_step.CLIP_LO, ref_step.CLIP_HI
        inP = ((sp >= lo) & (sp <= hi)).double()
        pe = torch.exp(sp.clamp(lo, hi))
        D = w * torch.exp(sn.clamp(lo, hi)).sum(0) + pe
        mag_pos = inP * (pe / D + 1.0)
    elif name == "self_adversarial":
        m, a = lp.get("margin", 3.0), lp.get("alpha", 0.5)
        p = torch.softmax(a * sn, dim=0)
        lj = torch.nn.functional.logsigmoid(-sn - m)
        S = (p * lj).sum(0, keepdim=True)
        mag_neg = w * p * (torch.sigmoid(sn + m) + a * (lj.abs() + S.abs()))
    return mag_pos, mag_neg


# --------------------------------------------------------------------------
# the step
# --------------------------------------------------------------------------
def oracle_step(model, ent, rel, triples, eta, neg_ent, neg_keep, loss="pairwise", loss_params=None, dpos=None,
                dneg=None, device="cpu", dtype=torch.float64, chunk=None, max_rel_size=None):
    """One step's scores, loss and gradient tables.  triples [B, 3]; neg_ent / neg_keep [eta*B], row j*B + i the j-th
    corruption of positive i (neg_keep = 1: the subject is kept, the object replaced).  dpos [B] / dneg [eta*B]: an
    external dL/dscore (KGE_STEP_BACKWARD_EXT) instead of the loss.  chunk: positives per autograd pass (the gradients
    of the loss, a sum over positives, are summed over the passes).  dtype float32 evaluates the same graph in fp32.
    -> Step of tensors on `device` (loss None with an external dL/dscore; sn, dsn, mag_neg as [eta*B])."""
    lp = dict(loss_params or {})
    dev = torch.device(device)
    E = torch.as_tensor(np.asarray(ent), dtype=dtype, device=dev).clone().requires_grad_(True)
    R = torch.as_tensor(np.asarray(rel), dtype=dtype, device=dev).clone().requires_grad_(True)
    mrs = max_rel_size or R.shape[0]
    t = torch.as_tensor(np.asarray(triples), dtype=torch.long, device=dev)
    B = t.shape[0]
    if neg_keep is None:  # neg_ent holds the corruption triples [eta*B, 3] themselves (e.g. the Philox draw)
        given = torch.as_tensor(np.asarray(neg_ent), dtype=torch.long, device=dev).reshape(eta, B, 3)
    else:
        ne = torch.as_tensor(np.asarray(neg_ent), dtype=torch.long, device=dev).reshape(eta, B)
        nk = torch.as_tensor(np.asarray(neg_keep), dtype=torch.long, device=dev).reshape(eta, B)
    if dpos is not None:
        dpos = torch.as_tensor(np.asarray(dpos), dtype=dtype, device=dev)
        dneg = torch.as_tensor(np.asarray(dneg), dtype=dtype, device=dev).reshape(eta, B)
    chunk = chunk or max(B, 1)
    loss_total = 0.0
    out = {k: [] for k in ("sp", "sn", "dsp", "dsn", "mp", "mn", "corr")}
    for a in range(0, B, chunk):
        b = min(B, a + chunk)
        tc = t[a:b]
        if neg_keep is None:
            corr = given[:, a:b].reshape(-1, 3)
        else:
            corr = ref_step.corrupt(tc, eta, nk[:, a:b].reshape(-1), ne[:, a:b].reshape(-1))
        sp = scores(model, E[tc[:, 0]], R[tc[:, 1]], E[tc[:, 2]], mrs)
        sn = scores(model, E[corr[:, 0]], R[corr[:, 1]], E[corr[:, 2]], mrs).reshape(eta, -1)
        if dpos is not None:
            dsp, dsn = dpos[a:b], dneg[:, a:b]
            obj = (sp * dsp).sum() + (sn * dsn).sum()
        else:
            obj = ref_step.per_positive_loss(loss, sp, sn, margin=lp.get("margin"), alpha=lp.get("alpha"),
                                             reduction=lp.get("reduction", "sum")).sum()
            dsp, dsn = torch.autograd.grad(obj, [sp, sn], retain_graph=True)
            loss_total += float(obj.detach())
        obj.backward()
        if dpos is None:
            mp, mn = loss_magnitudes(loss, sp, sn, lp, dsp, dsn)
        else:
            mp, mn = dsp.abs(), dsn.abs()
        for key, v in (("sp", sp), ("sn", sn), ("dsp", dsp), ("dsn", dsn), ("mp", mp), ("mn", mn), ("corr", corr)):
            out[key].append(v.detach())
    cat0 = lambda key: torch.cat(out[key], 0)
    cat1 = lambda key: torch.cat(out[key], 1).reshape(-1)
    corr = torch.cat([c.reshape(eta, -1, 3) for c in out["corr"]], 1).reshape(-1, 3)
    return Step(None if dpos is not None else loss_total, cat0("sp"), cat1("sn"), E.grad.detach(), R.grad.detach(),
                cat0("dsp"), cat1("dsn"), cat0("mp"), cat1("mn"), corr)


def grad_bound(model, ent, rel, triples, corr, mag_pos, mag_neg, device="cpu"):
    """Per-element inputs of the inexact-loss check, float64 on `device`: (A, A1, n) for the entity table and for the
    relation table.  A = sum_j mag_j |d score_j / d x| (the gradient of sum_j mag_j abs_scores_j on |tables|),
    A1 = sum_j |d score_j / d x|, n = the number of terms (lookups of the row in the step)."""
    dev = torch.device(device)
    Ea = torch.as_tensor(np.abs(np.asarray(ent)), dtype=torch.float64, device=dev).requires_grad_(True)
    Ra = torch.as_tensor(np.abs(np.asarray(rel)), dtype=torch.float64, device=dev).requires_grad_(True)
    t = torch.cat([torch.as_tensor(np.asarray(triples), dtype=torch.long, device=dev), corr.to(dev)], 0)
    mags = torch.cat([mag_pos.to(dev).double(), mag_neg.to(dev).double()])
    out = []
    for w in (mags, torch.ones_like(mags)):
        Ea.grad = Ra.grad = None
        (w * abs_scores(model, Ea[t[:, 0]], Ra[t[:, 1]], Ea[t[:, 2]])).sum().backward()
        out.append((Ea.grad.detach().clone(), Ra.grad.detach().clone()))
    n_e = torch.bincount(torch.cat([t[:, 0], t[:, 2]]), minlength=Ea.shape[0]).double()[:, None]
    n_r = torch.bincount(t[:, 1], minlength=Ra.shape[0]).double()[:, None]
    return (out[0][0], out[1][0], n_e), (out[0][1], out[1][1], n_r)


def within_bound(got, want, A, A1, n, extra):
    """|got - want| <= (n + 8 + extra) 2^-24 A + 2^-126 A1 per element (extra: the loss's own rounding chain).
    -> (ok, worst ratio of error to bound)."""
    got = torch.as_tensor(got, dtype=torch.float64, device=want.device)
    bound = (n + 8 + extra) * FP32_EPS * A + FP32_TINY * A1
    err = (got - want).abs()
    ratio = torch.where(bound > 0, err / torch.where(bound > 0, bound, torch.ones_like(bound)),
                        torch.where(err > 0, torch.full_like(err, float("inf")), torch.zeros_like(err)))
    return bool((err <= bound).all()), float(ratio.max()) if ratio.numel() else 0.0


def zipf_triples(E, R, n, rng):
    """s, o ~ truncated Zipf(1.0) over a random permutation of the entities (the GPU tests' positives)."""
    w = 1.0 / np.arange(1, E + 1)
    cdf = np.cumsum(w / w.sum())
    perm = rng.permutation(E)
    s, o = perm[np.searchsorted(cdf, rng.random(n))], perm[np.searchsorted(cdf, rng.random(n))]
    return np.stack([s, rng.integers(0, R, n), o], 1).astype(np.int32)
