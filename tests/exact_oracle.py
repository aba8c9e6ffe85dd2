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

For the 1vsAll family (1vsAll, KvsAll, relation prediction), whose every gradient element sums one term per (query,
candidate) pair, OvaBound gives the per-element bound in the same form, with each pair's weight derived in its
docstring from the kernels' split geometry (ova_chains) and the pair's logit error.

RotatE's training arithmetic is not exact on any grid (approximate sqrt / rsqrt, fp32 cos / sin): oracle_step(...,
rot_table=True) evaluates it on the rotation table the kernels read, and RotatEBound gives its per-element bound.

The predict path (kge_score_triples) has its own chain, one warp per triple: PredictBound gives its per-score bound.
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
    """sqrt(re^2 + im^2) whose gradient is 0 where the modulus is 0 (the reference's is NaN there).  The kernel's rot_unit
    (kge_train_common.cuh) takes g v rsqrt(max(|v|^2, 2^-126)): g v / |v| for |v|^2 >= 2^-126, g v 2^63 (at most |g|
    per component, 0 at an exactly zero residual) below; RotatEBound charges those terms in full."""

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


def rotation_divisor32(K, max_rel_size):
    """(div, inv_div) as the kernels have them: fp32(range / pi) (kge_create, kgeo_rotate_divisor) and fp32(1 / div)."""
    div = np.float32(ref_step.rotate_divisor(K, max_rel_size))
    return div, np.float32(1.0) / div


def rotation_table(theta, div):
    """(c, sn): the fp32 cos and sin of fp32(theta / div) by the canonical sincos -- the rotation table
    kge_rotation_table_kernel computes with kge_sincosf (kgeo_sincosf in the C oracle; pinned bit for bit by
    test_gpu_parity.py::test_corruption_scores_vs_oracle).  numpy float32 arrays of theta's shape."""
    from oracle import c_oracle
    phi = np.asarray(theta, np.float32) / np.float32(div)
    uniq, inv = np.unique(phi, return_inverse=True)
    s, c = c_oracle.sincos(uniq)
    return c[inv].reshape(phi.shape), s[inv].reshape(phi.shape)


class _KernelRotation(torch.autograd.Function):
    """theta -> (c, sn) of rotation_table, whose derivative is inv_div (-sn, c): the kernels' relation gradient
    fp32(1 / div) df/dphi, formed from the table's own values."""

    @staticmethod
    def forward(ctx, theta, div, inv_div):
        c, sn = rotation_table(theta.detach().cpu().numpy(), div)
        c = torch.as_tensor(c, dtype=theta.dtype, device=theta.device)
        sn = torch.as_tensor(sn, dtype=theta.dtype, device=theta.device)
        ctx.save_for_backward(c, sn)
        ctx.inv_div = float(inv_div)
        return c, sn

    @staticmethod
    def backward(ctx, gc, gs):
        c, sn = ctx.saved_tensors
        return ctx.inv_div * (c * gs - sn * gc), None, None


def scores(model, e_s, e_p, e_o, max_rel_size=None, rot_table=False):
    """ref_step.compute_scores, but RotatE's modulus through _Modulus; rot_table: RotatE's (cos, sin) from the fp32
    rotation table (_KernelRotation) instead of float64 cos / sin of theta / div."""
    if model != "RotatE":
        return ref_step.compute_scores(model, e_s, e_p, e_o, max_rel_size)
    h = e_s.shape[1] // 2
    theta = e_p[:, :h]
    if rot_table:
        p_re, p_im = _KernelRotation.apply(theta, *rotation_divisor32(e_s.shape[1], max_rel_size or 1))
    else:
        div = ref_step.rotate_divisor(e_s.shape[1], max_rel_size if max_rel_size else 1)
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
    assert model != "RotatE", "RotatE's bound is RotatEBound"
    h = e_s.shape[1] // 2
    s_re, s_im, p_re, p_im, o_re, o_im = e_s[:, :h], e_s[:, h:], e_p[:, :h], e_p[:, h:], e_o[:, :h], e_o[:, h:]
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
                dneg=None, device="cpu", dtype=torch.float64, chunk=None, max_rel_size=None, rot_table=False):
    """One step's scores, loss and gradient tables.  triples [B, 3]; neg_ent / neg_keep [eta*B], row j*B + i the j-th
    corruption of positive i (neg_keep = 1: the subject is kept, the object replaced).  dpos [B] / dneg [eta*B]: an
    external dL/dscore (KGE_STEP_BACKWARD_EXT) instead of the loss.  chunk: positives per autograd pass (the gradients
    of the loss, a sum over positives, are summed over the passes).  dtype float32 evaluates the same graph in fp32.
    rot_table: RotatE on the kernels' fp32 rotation table (scores).
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
        sp = scores(model, E[tc[:, 0]], R[tc[:, 1]], E[tc[:, 2]], mrs, rot_table)
        sn = scores(model, E[corr[:, 0]], R[corr[:, 1]], E[corr[:, 2]], mrs, rot_table).reshape(eta, -1)
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


def within_bound(got, want, A, A1, n, extra, absolute=0.0):
    """|got - want| <= (n + 8 + extra) 2^-24 A + 2^-126 A1 + absolute per element (extra: the loss's own rounding
    chain; absolute: per-term allowances that are not a multiple of A, RotatEBound's).
    -> (ok, worst ratio of error to bound)."""
    got = torch.as_tensor(got, dtype=torch.float64, device=want.device)
    bound = (n + 8 + extra) * FP32_EPS * A + FP32_TINY * A1 + absolute
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


# --------------------------------------------------------------------------
# RotatE: a per-element bound
# --------------------------------------------------------------------------
# The MUFU approximations of the RotatE training kernels (kge_train_common.cuh: sqrt_approx, rsqrt_approx), from the
# PTX ISA's instruction descriptions: sqrt.approx.f32 has a maximum relative error of 2^-23 and rsqrt.approx.f32 one of
# 2^-22.9 over the range of normal inputs (the .ftz forms flush subnormal inputs to 0).  scripts/check_sqrt.cu measures
# both over every normal float: 2^-23.25 and 2^-22.94 on an H100 80GB HBM3 at 700 W (DESIGN.md 3.4).
EPS_SQRT = 2.0 ** -23
EPS_RSQ = 2.0 ** -22.9
ROT_C = 8  # roundings of one gradient element outside the term sums: back-rotation (2), inv_div (1), the Z / Aphi fma


def loss_chain(loss, lp, sp, sn):
    """Per score of each positive ([eta+1, B], row 0 the positive): c such that the rounding of the kernels' loss chain
    (loss_and_dscores, kge_train_common.cuh, built without fast math) moves its dL/dscore by at most c u mag
    (loss_magnitudes), u = 2^-24.  Library maths (CUDA C Programming Guide, Mathematical Functions): expf 2 ulp (4u),
    logf / log1pf 1 ulp (2u); x / y is the IEEE quotient (1u); w = fl(1 / eta) and w2 = fl(1 / (2 eta)) 1u each (2 eta
    is exact).  A sum of m nonzero terms in any order (lane loops, warp sums: adds of exact zeros are exact) rounds each
    term at most m - 1 times.  In units of u:
      pairwise:        dN = w (1), dP = -(sum of eta copies of w) (eta);  absolute_margin: dP = -w eta (2).
      nll:             q = e / (1 + e): e 4, 1 + e 5, quotient 1 -> 10; dN = (w2 inN) q: 12; dP = -w2 eta inP q: 13.
      multiclass_nll:  D = w sum_j e_j + pe: e_j 4, the sum eta - 1, w and its product 2, the add 1 -> eta + 6;
                       dN = ((w inN) e_j) / D: eta + 13; dP = inP (pe / D - 1): eta + 11, then 1 relative to
                       pe / D + 1 (mag_pos) -> eta + 12.
      -> 2 eta + 16 covers these three (and nll's 13).
      self_adversarial (both code paths, eta <= 32 and the looped one): with A = max_j (alpha |N_j| + |alpha N_j - mx|)
        (the rounding of exp's argument alpha N - mx, amplified by exp into a relative error) and X = max(|P + m|,
        max_j |N_j + m|) (that of x = -N - m, and of the positive's m + P), e_j: 4 + A; z: eta - 1 + 4 + A;
        p_j = e_j / z: eta + 8 + 2A; t = exp(-|x|): 4 + X; log1p(t): (6 + X) log1p(t) since t / (1 + t) <= log1p(t);
        l_j = min(x, 0) - log1p(t): (7 + X) |l_j| (both parts have the sign of l_j); sg_j: 10 + 2X; S = sum p l:
        (2 eta + 7 + 2 (4 + A) + X) |S| (all l_j <= 0, so |S| = sum p |l|); pj sg: eta + 19 + 2A + 2X;
        alpha pj (l_j - S): (3 eta + 26 + 4A + X) (|l_j| + |S|); the difference, w and its product 3 more:
        -> 3 eta + 30 + 4A + 2X relative to mag_neg = w p (sg + alpha (|l| + |S|)); dP = -1 / (1 + exp(m + P)): 6 + X."""
    sp, sn = sp.detach(), sn.detach()
    eta = sn.shape[0]
    c = torch.full((eta + 1, sp.shape[0]), float(2 * eta + 16), dtype=torch.float64, device=sp.device)
    if loss == "self_adversarial":
        lp = dict(lp or {})
        m, a = lp.get("margin", 3.0), lp.get("alpha", 0.5)
        an = a * sn
        A = (an.abs() + (an - an.max(0, keepdim=True).values).abs()).max(0).values
        X = torch.maximum((sp + m).abs(), (sn + m).abs().max(0).values)
        c = (3 * eta + 30 + 4 * A + 2 * X)[None].expand(eta + 1, -1).clone()
    return c


def loss_premises(loss, lp, sp, sn, dsp_err, dsn_err):
    """The data's premises for a fused step whose scores are off by up to dsp_err / dsn_err: no hinge argument of
    pairwise (m - P + N, two roundings of at most u (|m| + |P| + |N|) on top of the score errors) or absolute_margin
    (m + N, one rounding, which keeps the sign) lies within its error of 0, where dL/dscore jumps; no clipped loss's
    (nll, multiclass_nll) score lies within its error of +-75, where the clip mask flips.  Asserted, not assumed."""
    lp = dict(lp or {})
    u = FP32_EPS
    if loss in ("pairwise", "absolute_margin"):
        mg = lp.get("margin", 1.0)
        if loss == "pairwise":
            arg = mg - sp[None] + sn
            err = dsn_err + dsp_err[None] + 2 * u * (1 + 2 * u) * (abs(mg) + sp.abs()[None] + sn.abs())
        else:
            arg, err = mg + sn, dsn_err
        assert not bool((arg.abs() <= err).any()), "premise: a hinge argument lies within its score bound of 0"
    if loss in ("nll", "multiclass_nll"):
        for s, e in ((sp, dsp_err), (sn, dsn_err)):
            assert not bool(((s.abs() - ref_step.CLIP_HI).abs() <= e).any()), "premise: a score within its bound of 75"


def loss_error(loss, lp, step, eta, dsp_err, dsn_err, device):
    """dL/dscore error and loss error of a fused step whose scores are off by up to dsp_err [B] / dsn_err [eta, B],
    shared by RotatEBound and TrilinearBound.  -> (dg [B + eta*B] in step's score order, loss_err).
      dg_j = sum_i |H_ji| ds_i (loss_score_sensitivity: the positive's Hessian block, first order) + c_j u mag_j
      (loss_chain); loss None (KGE_STEP_BACKWARD_EXT): the given dL/dscore is exact, dg = 0.
      The loss: per positive sum_j |g_j| ds_j + (c + 16) u (|L_i| + sum_j |g_j| (|s_j| + |margin|) + eta + 1), c the
      positive's largest chain: each of its eta + 1 loss terms phi is evaluated with at most c roundings relative to
      |phi|, to its argument (|phi'| |s + margin|, and |phi'| = |g| / w is carried by the loss's own factor w) and to 1
      (logf / log1pf of a quantity near 1 err by a unit absolute), then summed (eta more) and accumulated in fp64."""
    u = FP32_EPS
    B = dsp_err.shape[0]
    if loss is None:
        return torch.zeros(B * (eta + 1), dtype=torch.float64, device=device), 0.0
    lp = dict(lp or {})
    sp, snn = step.sp.to(device).double(), step.sn.to(device).double().reshape(eta, B)
    loss_premises(loss, lp, sp, snn, dsp_err, dsn_err)
    hp, hn = loss_score_sensitivity(loss, lp, sp, snn, dsp_err, dsn_err)
    c = loss_chain(loss, lp, sp, snn)
    mag = torch.cat([step.mag_pos.to(device).double()[None], step.mag_neg.to(device).double().reshape(eta, B)], 0)
    dg = torch.cat([hp, hn.reshape(-1)]) + u * torch.cat([(c * mag)[0], (c * mag)[1:].reshape(-1)])
    gl = torch.cat([step.dsp[None], step.dsn.reshape(eta, B)], 0).to(device).double().abs()
    sc = torch.cat([sp[None], snn], 0).abs()
    err = torch.cat([dsp_err[None], dsn_err], 0)
    mg = abs(lp.get("margin", 3.0 if loss == "self_adversarial" else 1.0))
    loss_err = float((gl * err).sum() + (u * (c.max(0).values + 16) * (gl * (sc + mg)).sum(0)).sum()
                     + (c.max(0).values + 16).max() * u * (abs(step.loss) + (eta + 1) * B))
    return dg, loss_err


def loss_score_sensitivity(loss, lp, sp, sn, dsp_err, dsn_err):
    """Per score j of each positive: sum_i |d^2 L / d s_j d s_i| ds_i over the positive's eta + 1 scores (the
    (eta+1)^2 Hessian block of per_positive_loss, float64 autograd): how far a score error ds moves dL/dscore.
    sp [B], sn [eta, B] -> ([B], [eta, B]).  The hinge losses' Hessian is 0 (see RotatEBound for their premise)."""
    lp = dict(lp or {})
    s = torch.cat([sp.detach()[None], sn.detach()], 0).clone().requires_grad_(True)
    err = torch.cat([dsp_err[None], dsn_err], 0)
    L = ref_step.per_positive_loss(loss, s[0], s[1:], margin=lp.get("margin"), alpha=lp.get("alpha"),
                                   reduction=lp.get("reduction", "sum")).sum()
    G = torch.autograd.grad(L, s, create_graph=True)[0]
    out = torch.zeros_like(err)
    if G.requires_grad:
        for k in range(s.shape[0]):  # row k of every positive's block at once (the blocks do not interact)
            Hk = torch.autograd.grad(G[k].sum(), s, retain_graph=True, allow_unused=True)[0]
            if Hk is not None:
                out[k] = (Hk.abs() * err).sum(0)
    return out[0], out[1:]


class RotatEBound:
    """The per-element error bound of one RotatE training step (kge_train_rot_kernel and the general kernel's RotatE
    Scorer, which share the rot_* functions of kge_train_common.cuh), against oracle_step(..., rot_table=True): both
    read the same fp32 rotation table (c, sn), so the bound covers the training arithmetic only.  u = 2^-24.

    Every score row j (positive or corruption; x its subject-slot row, o its object-slot row, g_j = dL/dscore_j) adds,
    per complex column d, one term to each of x's two elements, o's two and theta_d.  With y = R(phi) x, v = y - o,
    m = |v| and U = g v / m:  d/do = U,  d/dx = -R(-phi) U,  d/dtheta = inv_div (U_re y_im - U_im y_re).
      * Residual.  Object-slot chains rot_rotate then a subtraction (the gradient pass, and the score pass of the
        positive and of object-replaced rows), or rot_residual_subj (two dependent fmas; score pass of subject-
        replaced rows).  Either way each component is within 3 u S_c (1 + 2u) + 2^-125 of the exact one, S_re = |x_re c|
        + |x_im sn| + |o_re|, S_im = |x_re sn| + |x_im c| + |o_im| (two or three roundings, each at most u times a
        partial sum bounded by S_c; 2^-125 for flushed subnormal intermediates).  dv = delta_re + delta_im >= |dv|.
      * Unit vector.  rot_unit forms |v|^2 = fma(im, im, re re) (2u relative, plus 2^-125 absolute when squares fall
        below 2^-126), rsqrt.approx (EPS_RSQ) and two products (2u): every component of the kernel's (a, b) is within
            E = |g| min(2 dv / m + EPS_RSQ + 4u + 2^-125 / m^2,  2 + EPS_RSQ + 4u) + |dg| (1 + EPS_RSQ + 4u)
        of U's, dg the error of g.  2 dv / m bounds |v/|v| - v'/|v'|| for |v - v'| <= dv; it is ill-conditioned as m
        -> 0 and is carried per term.  The cap holds because both vectors have norm at most |g| (1 + EPS_RSQ + 4u); it
        also covers |v|^2 < 2^-126, where rot_unit returns g v 2^63 (at most |g| per component).
      * Terms.  Per element the term's magnitude w and its absolute allowance X are: o's elements w = |g|, X = E;
        x's elements w = |g| (|c| + |sn|), X = E (|c| + |sn|); theta_d w = inv_div |g| (|y_re| + |y_im|),
        X = inv_div (E (|y_re| + |y_im|) + |g| dy), dy = 2u (|x_re c| + |x_im sn| + |x_re sn| + |x_im c|) the error of
        the kernel's y.  A = sum of w, absolute = sum of X.
      * Sums.  The register sums Z* / Aphi (up to eta + 1 terms, summed before the back-rotation in finish), the
        back-rotation and the red.global.add atomics in any order: (n + 8 + ROT_C) u A with n = the element's lookups
        + eta + 2; the atomics flush subnormal results, 2^-126 each (A1 = n + 8).
      * Scores.  |delta s| <= sum_d (dv_d + (m_d + dv_d)(EPS_SQRT + 2u)) + (h + 16) u sum_d (m_d + dv_d) + h 2^-62:
        the residual, |v|^2's rounding (2u relative, half of it through the sqrt) and sqrt.approx, the sum of h moduli
        (float4 sums, fma with the lane mask, warp sum), and sqrt.approx.ftz flushing |v|^2 < 2^-126 to 0
        (sqrt(2^-125) < 2^-62).
      * Fused losses and the loss value: loss_error (shared with TrilinearBound).  dg_j = sum_i |H_ji| delta s_i (the
        positive's Hessian block) plus the loss chain's own roundings (loss_chain).  For pairwise and absolute_margin
        the Hessian is 0 away from the hinge, so the data must keep every hinge argument farther than its error from 0
        (loss_premises: asserted, a premise of the data, not a property of the kernel).
    loss None: KGE_STEP_BACKWARD_EXT (g given and exact, dg = 0)."""

    def __init__(self, ent, rel, triples, step, eta, loss=None, loss_params=None, max_rel_size=None, device="cpu"):
        u = FP32_EPS
        dev = self.device = torch.device(device)
        E = torch.as_tensor(np.asarray(ent), dtype=torch.float64, device=dev)
        R = torch.as_tensor(np.asarray(rel), dtype=torch.float64, device=dev)
        K = E.shape[1]
        h = K // 2
        div, inv_div = rotation_divisor32(K, max_rel_size or R.shape[0])
        inv_div = float(inv_div)
        ct, st = rotation_table(np.asarray(rel, np.float32)[:, :h], div)
        ct = torch.as_tensor(ct, dtype=torch.float64, device=dev)
        st = torch.as_tensor(st, dtype=torch.float64, device=dev)
        t = torch.as_tensor(np.asarray(triples), dtype=torch.long, device=dev)
        B = t.shape[0]
        T = torch.cat([t, step.corr.to(dev)], 0)
        g = torch.cat([step.dsp, step.dsn]).to(dev).double()
        X, O, c, sn = E[T[:, 0]], E[T[:, 2]], ct[T[:, 1]], st[T[:, 1]]
        xr, xi, orr, oi = X[:, :h], X[:, h:], O[:, :h], O[:, h:]
        yr, yi = xr * c - xi * sn, xr * sn + xi * c
        m = torch.sqrt((yr - orr) ** 2 + (yi - oi) ** 2)
        Sre = (xr * c).abs() + (xi * sn).abs() + orr.abs()
        Sim = (xr * sn).abs() + (xi * c).abs() + oi.abs()
        dv = 3 * u * (1 + 2 * u) * (Sre + Sim) + 2.0 ** -124
        mm = m + dv
        self.score_err = ((dv + mm * (EPS_SQRT + 2 * u)).sum(1) + (h + 16) * u * mm.sum(1) + h * 2.0 ** -62)
        dsp_err, dsn_err = self.score_err[:B], self.score_err[B:].reshape(eta, B)
        dg, self.loss_err = loss_error(loss, loss_params, step, eta, dsp_err, dsn_err, dev)
        ga, dga = g.abs()[:, None], dg[:, None]
        rel_e = torch.where(m > 0, 2 * dv / torch.where(m > 0, m, torch.ones_like(m)) + EPS_RSQ + 4 * u
                            + 2.0 ** -125 / torch.where(m > 0, m * m, torch.ones_like(m)), torch.full_like(m, np.inf))
        Eu = ga * torch.clamp(rel_e, max=2 + EPS_RSQ + 4 * u) + dga * (1 + EPS_RSQ + 4 * u)
        cs = c.abs() + sn.abs()
        ya = yr.abs() + yi.abs()
        dy = 2 * u * (Sre + Sim - orr.abs() - oi.abs())
        self.A = [torch.zeros_like(E), torch.zeros_like(R)]
        self.X = [torch.zeros_like(E), torch.zeros_like(R)]
        for rows, w, x in ((T[:, 0], ga * cs, Eu * cs), (T[:, 2], ga.expand(-1, h), Eu)):
            self.A[0].index_add_(0, rows, torch.cat([w, w], 1))
            self.X[0].index_add_(0, rows, torch.cat([x, x], 1))
        self.A[1][:, :h].index_add_(0, T[:, 1], inv_div * ga * ya)
        self.X[1][:, :h].index_add_(0, T[:, 1], inv_div * (Eu * ya + ga * (1 + 4 * u) * dy))
        n_e = torch.bincount(torch.cat([T[:, 0], T[:, 2]]), minlength=E.shape[0]).double()[:, None]
        n_r = torch.bincount(t[:, 1], minlength=R.shape[0]).double()[:, None]
        self.n = [n_e + eta + 2, n_r + eta + 2]

    def check(self, got_ent, got_rel, want_ent, want_rel):
        """-> [(name, ok, worst error / bound)] for both gradient tables."""
        out = []
        for i, (name, got, want) in enumerate((("g_ent", got_ent, want_ent), ("g_rel", got_rel, want_rel))):
            want = torch.as_tensor(want, dtype=torch.float64).to(self.device)
            got = torch.as_tensor(got, dtype=torch.float64).to(self.device)
            if not bool(torch.isfinite(got).all()):
                out.append((name, False, float("inf")))
                continue
            ok, ratio = within_bound(got, want, self.A[i], self.n[i] + 8, self.n[i], ROT_C, self.X[i])
            out.append((name, ok, ratio))
        return out

    def check_scores(self, got, want, which):
        """got / want [B] (which 'sp') or [eta*B] ('sn') -> (ok, worst error / bound)."""
        B = len(self.score_err) - len(want) if which == "sn" else 0
        bound = self.score_err[B:B + len(want)] if which == "sn" else self.score_err[:len(want)]
        got = torch.as_tensor(got, dtype=torch.float64).to(self.device)
        err = (got - torch.as_tensor(want, dtype=torch.float64).to(self.device)).abs()
        return bool((err <= bound).all()), float((err / bound).max()) if err.numel() else 0.0


# --------------------------------------------------------------------------
# DistMult, ComplEx, HolE and TransE: a per-element bound
# --------------------------------------------------------------------------
TRI_C = 5  # roundings of one gradient term outside its register and row sums (TrilinearBound)


def score_chain(model, K):
    """Roundings any one product (TransE: column) of a score passes through in the training kernels (TrilinearBound)."""
    halves = 1 if model in ("TransE", "DistMult") else 2
    kp = -(-(K // halves) // 4) * 4
    return halves * (-(-kp // 128) + -(-kp // 512)) + -(-kp // 512) + 11


class TrilinearBound:
    """The per-element error bound of one DistMult / ComplEx / HolE / TransE training step (the general kernel, the
    resident fast path kge_train_res_kernel in its scatter and GATHER forms, the bucket sum and the deferred owner
    kernel, which share the per-model functions of kge_train_common.cuh) against oracle_step in float64.  u = 2^-24;
    |.| of a term below is its value with every product counted positive (abs_scores on |tables|).
      * Scores.  A trilinear score is a sum of m products (DistMult m = k; ComplEx / HolE four per complex column).
        Each product carries: its query vector (query_subj / query_obj: pr * orr is one rounding, the ComplEx forms
        two: a product and an fma or a subtraction), the lane's fma chain into its float4 chunk sums (at most
        HALVES ceil(kp / 128) fmas, plus one per column window of the general kernel: HALVES ceil(kp / 512)), f4hsum
        (2), the warp sum (5 shuffle levels), the sum over column windows (ceil(kp / 512)), and HolE's scale: 2 / k is
        stored as fl(2 / k) (1, exact when k is a power of two) and multiplied in (1).  TransE: the residual s + p - o
        in two roundings (the residual has magnitude at most |s| + |p| + |o|, its sign is exact by the premise below),
        f4abssum (2), the lane chain, the warp sum.  So |delta s| <= score_chain u |s| + m 2^-149 (subnormal
        products), score_chain = HALVES (ceil(kp / 128) + ceil(kp / 512)) + ceil(kp / 512) + 11.
      * dL/dscore.  loss_error: the score errors through each positive's Hessian block, plus loss_chain (derived there:
        expf / logf / log1pf without fast math, w = 1 / eta and w2 = 1 / (2 eta), multiclass_nll's pe / D - 1 and
        self_adversarial's p_j (l_j - S)), under loss_premises (hinge arguments and clip bounds away from the kinks).
        KGE_STEP_BACKWARD_EXT: g is given and exact, dg = 0.
      * Gradient elements.  Element x of a row is sum_j g_j d s_j / d x.  The kernel scales g by fl(2 / k) for HolE
        (2 roundings, 0 otherwise).  A replaced row's term is g * Q (Q: 2, the product: 1).  The kept rows are formed
        in factored form: U = gP s + sum_j g_j r_j (and X for the object slot) is a register sum of eta + 1 fmas, then
        query_subj / query_obj (2) or trilinear_grad_p (3: two products / fmas and the final add); TransE sums
        g_j sign(residual) (exact by the premise) over eta + 1 terms and adds the kept shares (2 adds).  So each term
        passes through at most TRI_C = 5 roundings of its own and eta + 1 register adds.  The row's contributions (one
        per positive lookup: the kept rows' REDs or hot-entity registers; one per replaced lookup: REDs, bucket runs, the
        owner kernel's grad[e] + sum) are summed in some order with at most n - 1 adds, n the row's positive lookups
        plus its replaced lookups (a corruption's kept side is folded into its positive's register sum).  With g's error dg (|g + dg| <= mag + dg, loss_magnitudes):
            |err| <= (n + eta + 2 + 8 + TRI_C) u sum_j (mag_j + dg_j) |d s_j / d x| + sum_j dg_j |d s_j / d x|
                     + 2^-126 (n + eta + 10)
        (within_bound with A = grad_bound(mag + dg), absolute = grad_bound(dg)).  The 8 covers the second-order terms:
        (1 + u)^N - 1 - N u <= N^2 u^2 / (1 - N u) <= 8 u for N <= 11,000 (asserted); 2^-126 per add for the
        atomics' and sums' flushed subnormal results.
      * Premise of TransE: no residual s + p - o lies within 2 u (1 + u) (|s| + |p| + |o|) of 0, where |x|' jumps
        (asserted on the data).
      * Loss: loss_error."""

    def __init__(self, model, ent, rel, triples, step, eta, loss=None, loss_params=None, device="cpu"):
        assert model in TRILINEAR + ("TransE",)
        u = FP32_EPS
        dev = self.device = torch.device(device)
        E = torch.as_tensor(np.asarray(ent), dtype=torch.float64, device=dev)
        R = torch.as_tensor(np.asarray(rel), dtype=torch.float64, device=dev)
        K = E.shape[1]
        t = torch.as_tensor(np.asarray(triples), dtype=torch.long, device=dev)
        B = t.shape[0]
        T = torch.cat([t, step.corr.to(dev)], 0)
        Ea, Ra = E.abs(), R.abs()
        asc = abs_scores(model, Ea[T[:, 0]], Ra[T[:, 1]], Ea[T[:, 2]])
        m = K if model in ("TransE", "DistMult") else 2 * K
        self.score_err = score_chain(model, K) * u * asc + m * 2.0 ** -149
        if model == "TransE":
            for a in range(0, T.shape[0], 1 << 16):
                Tc = T[a:a + (1 << 16)]
                res = E[Tc[:, 0]] + R[Tc[:, 1]] - E[Tc[:, 2]]
                tol = 2 * u * (1 + 2 * u) * (Ea[Tc[:, 0]] + Ra[Tc[:, 1]] + Ea[Tc[:, 2]])
                assert not bool((res.abs() <= tol).any()), "premise: a TransE residual lies within its rounding of 0"
        dsp_err, dsn_err = self.score_err[:B], self.score_err[B:].reshape(eta, B)
        dg, self.loss_err = loss_error(loss, loss_params, step, eta, dsp_err, dsn_err, dev)
        mag = torch.cat([step.mag_pos, step.mag_neg]).to(dev).double() + dg
        (A0, _, _), (A1, _, _) = grad_bound(model, ent, rel, triples, step.corr, mag[:B], mag[B:], dev)
        (X0, _, _), (X1, _, _) = grad_bound(model, ent, rel, triples, step.corr, dg[:B], dg[B:], dev)
        self.A, self.X = [A0, A1], [X0, X1]
        # a row's contributions: one per positive lookup (the kept rows' register sums) and one per replaced lookup
        tc = T[B:]
        repl = torch.where(tc[:, 0] != t[:, 0].repeat(eta), tc[:, 0], tc[:, 2])
        n_e = torch.bincount(torch.cat([t[:, 0], t[:, 2], repl]), minlength=E.shape[0]).double()[:, None]
        n_r = torch.bincount(t[:, 1], minlength=R.shape[0]).double()[:, None]
        self.n = [n_e + eta + 2, n_r + eta + 2]
        assert max(float(n.max()) for n in self.n) + 8 + TRI_C <= 11000, "second-order allowance"

    def check(self, got_ent, got_rel, want_ent, want_rel):
        """-> [(name, ok, worst error / bound)] for both gradient tables."""
        out = []
        for i, (name, got, want) in enumerate((("g_ent", got_ent, want_ent), ("g_rel", got_rel, want_rel))):
            want = torch.as_tensor(want, dtype=torch.float64).to(self.device)
            got = torch.as_tensor(got, dtype=torch.float64).to(self.device)
            if not bool(torch.isfinite(got).all()):
                out.append((name, False, float("inf")))
                continue
            ok, ratio = within_bound(got, want, self.A[i], self.n[i] + 8, self.n[i], TRI_C, self.X[i])
            out.append((name, ok, ratio))
        return out

    check_scores = RotatEBound.check_scores


# --------------------------------------------------------------------------
# kge_score_triples (the predict path): a per-element bound
# --------------------------------------------------------------------------
def predict_chain(model, k):
    """N: the roundings any one product (TransE and RotatE: column term) of a predict score passes through (PredictBound),
    L = ceil(k / 32) columns per lane."""
    L = -(-k // 32)
    return {"DistMult": 1 + L + 5, "ComplEx": 2 + 2 * L + 5, "HolE": 2 + 2 * L + 5 + 2, "TransE": 2 + L + 5,
            "RotatE": 5 + L + 5}[model]


def predict_abs(model, e_s, e_p, e_o, c=None, sn=None):
    """Per triple, the magnitude PredictBound's relative term scales: abs_scores on |tables| (HolE's exact 2 / k
    included); RotatE sum_d S_re + S_im with (c, sn) the rotation-table row, S_re = |s_re c| + |s_im sn| + |o_re|,
    S_im = |s_re sn| + |s_im c| + |o_im|."""
    if model != "RotatE":
        return abs_scores(model, e_s.abs(), e_p.abs(), e_o.abs())
    h = e_s.shape[1] // 2
    sr, si, o = e_s[:, :h].abs(), e_s[:, h:].abs(), e_o.abs()
    c, sn = c.abs(), sn.abs()
    return (sr * (c + sn) + si * (sn + c)).sum(1) + o.sum(1)


def nonfinite_class(x):
    """0 finite, 1 NaN, 2 +inf, 3 -inf, elementwise (float64 tensor)."""
    cls = torch.zeros(x.shape, dtype=torch.int8, device=x.device)
    cls[torch.isnan(x)] = 1
    cls[x == np.inf] = 2
    cls[x == -np.inf] = 3
    return cls


class PredictBound:
    """The per-element error bound of kge_score_triples (kge_misc.cu: kge_score_kernel, the predict path), against
    scores(..., rot_table=True) in float64 on the fp32 tables: RotatE reads the kernels' fp32 rotation table (c, sn)
    on both sides (pinned bit for bit elsewhere), so the bound covers the scoring arithmetic only.  u = 2^-24.

    One warp per triple: lane l accumulates columns l, l + 32, ... < k (L = ceil(k / 32) of them) in one fp32 register,
    warp_sum (an xor butterfly, 5 levels) adds the 32 lanes, lane 0 stores scale * acc (scale = fl(2 / k) for HolE, 1
    otherwise).  The library is built without fast math (kge_misc.cu's PTX: sqrt.rn.f32, no .ftz, no .approx), and
    --fmad=true contracts nothing here: every product feeds an explicit fmaf, a store or a multiply.  A sum evaluated in
    any order rounds each term once per add it passes through (relative to the sum of the terms' magnitudes), so it
    is enough to count, per product, the roundings on its way to the output:
      DistMult   acc = fmaf(s * p, o, acc): s * p (1), the lane's L fmas (the first one adds to an exact 0, still at
                 most L), the butterfly (5)                                                  N = 1 + L + 5.
      ComplEx    acc = fmaf(sr, fmaf(pi, oi, pr * orr), acc), then fmaf(si, fmaf(-pi, orr, pr * oi), acc): the inner
                 product and fma (2; 1 for the fma's own product), 2L outer fmas, the butterfly   N = 2 + 2L + 5.
      HolE       ComplEx's chain, then scale = fl(2 / k) (1, exact when k is a power of two) and the multiply (1):
                                                                                              N = 2 + 2L + 5 + 2.
      TransE     acc -= fabsf((s + p) - o): the residual's two adds are within ((1 + u)^2 - 1)(|s| + |p| + |o|) of
                 the exact one and fabsf is 1-Lipschitz, so |s| + |p| + |o| carries it (no premise on the residual's
                 sign); L subtractions, the butterfly                                         N = 2 + L + 5.
      RotatE     re = fmaf(-si, sn, sr * c) - o_re: s_re c passes 3 roundings, s_im sn 2, o_re 1, so |re' - re| <=
                 ((1 + u)^3 - 1) S_re, and the same for im with S_im; the modulus is 1-Lipschitz in (re, im), so
                 |m' - m| <= ((1 + u)^3 - 1) S, S = S_re + S_im (predict_abs).  sqrtf(fmaf(im, im, re * re)): the sum
                 of squares is within (1 + u)^2 of re'^2 + im'^2, its square root within (1 + u) and sqrt.rn another
                 (1 + u), so 2 more relative to m' <= S (1 + u)^3; then L subtractions and the butterfly.  N = 5 + L + 5.
    So |got - want| <= ((1 + u)^N - 1) A <= (N + 1) u A with A = predict_abs; the + 1 is the second-order term:
    (1 + u)^N - 1 - N u <= N^2 u^2 / (1 - N u) <= u for N <= 4,095 (asserted).
    Underflow.  A rounding to a subnormal result adds at most 2^-150 absolute; adds and subtractions whose result is
    subnormal are exact.  DistMult has 2 products / fmas per column that can underflow, ComplEx and HolE 6, TransE none;
    each such error is then scaled by at most scale (1 + u)^(N + 2) < 4 (scale <= 2 at k = 1), and HolE's final multiply
    adds one more: (n_u + 1) 2^-148 per triple, n_u = 2k, 6k or 0.  RotatE: the products of the residual and the
    square re' * re' and the fma can underflow, which moves the sum of squares by at most 2^-148.9 absolute; through the
    square root that is sqrt(2^-148.9) < 2^-74.4, so 2^-74 per column (the residual's own 2^-148 included): h 2^-74.
    Non-finite entries: where a row holds +-inf or NaN and no finite value overflows, the score is NaN, +inf or -inf
    exactly where the float64 oracle's is (every non-finite product term meets the same sums in any order: NaN is
    absorbing and +inf + -inf is NaN); check compares these classes exactly."""

    def __init__(self, model, ent, rel, triples, max_rel_size=None, device="cpu", chunk=1 << 12):
        u = FP32_EPS
        self.model, dev = model, torch.device(device)
        self.device = dev
        E = torch.as_tensor(np.asarray(ent), dtype=torch.float64, device=dev)
        R = torch.as_tensor(np.asarray(rel), dtype=torch.float64, device=dev)
        self.t = t = torch.as_tensor(np.asarray(triples), dtype=torch.long, device=dev).reshape(-1, 3)
        K = E.shape[1]
        k = K if model in ("TransE", "DistMult") else K // 2
        self.mrs = max_rel_size or R.shape[0]
        N = predict_chain(model, k)
        assert N <= 4095, "second-order allowance"
        if model == "RotatE":
            ct, st = rotation_table(np.asarray(rel, np.float32)[:, :k], rotation_divisor32(K, self.mrs)[0])
            ct = torch.as_tensor(ct, dtype=torch.float64, device=dev)
            st = torch.as_tensor(st, dtype=torch.float64, device=dev)
            absolute = k * 2.0 ** -74
        else:
            absolute = ({"DistMult": 2 * k, "ComplEx": 6 * k, "HolE": 6 * k, "TransE": 0}[model] + 1) * 2.0 ** -148
        want, bound = [], []
        with np.errstate(all="ignore"):
            for a in range(0, t.shape[0], chunk):
                tc = t[a:a + chunk]
                s, p, o = E[tc[:, 0]], R[tc[:, 1]], E[tc[:, 2]]
                want.append(scores(model, s, p, o, self.mrs, rot_table=True))
                rot = dict(c=ct[tc[:, 1]], sn=st[tc[:, 1]]) if model == "RotatE" else {}
                bound.append((N + 1) * u * predict_abs(model, s, p, o, **rot) + absolute)
        self.want = torch.cat(want) if want else torch.zeros(0, dtype=torch.float64, device=dev)
        self.bound = torch.cat(bound) if bound else torch.zeros(0, dtype=torch.float64, device=dev)

    def check(self, got, want=None, rows=None):
        """got [n] (or [len(rows)] with rows: indices into the triples) against want (default the oracle's scores):
        the non-finite classes equal and every finite element within the bound.  -> (ok, worst error / bound over
        the finite elements, index of the worst element (of rows, when given), or of the first class mismatch)."""
        got = torch.as_tensor(np.asarray(got), dtype=torch.float64).to(self.device)
        idx = slice(None) if rows is None else torch.as_tensor(np.asarray(rows), dtype=torch.long, device=self.device)
        want = self.want[idx] if want is None else torch.as_tensor(want, dtype=torch.float64).to(self.device)
        bound = self.bound[idx]
        cg, cw = nonfinite_class(got), nonfinite_class(want)
        if not bool((cg == cw).all()):
            return False, float("inf"), int(torch.nonzero(cg != cw)[0, 0])
        fin = cw == 0
        err = torch.where(fin, (got - want).abs(), torch.zeros_like(got))
        ratio = err / torch.where(fin, bound, torch.ones_like(bound))
        if ratio.numel() == 0:
            return True, 0.0, -1
        worst = int(ratio.argmax())
        return bool((err <= torch.where(fin, bound, torch.zeros_like(bound))).all()), float(ratio[worst]), worst

    def assert_within(self, got, where=""):
        """check, asserted with the worst element's triple, got, want and bound in the message.  -> worst ratio."""
        ok, ratio, i = self.check(got)
        if not ok:
            g = float(np.asarray(got, np.float64).reshape(-1)[i])
            raise AssertionError("%s: element %d, triple %s: got %r, want %r, bound %r (worst error / bound %.3g)" % (
                where, i, self.t[i].tolist(), g, float(self.want[i]), float(self.bound[i]), ratio))
        return ratio


# --------------------------------------------------------------------------
# engine plumbing shared by the GPU tests
# --------------------------------------------------------------------------
def dense(eng, table):
    """padded [rows, ld] -> dense [rows, internal_k] float64 on the host, and whether every pad column is 0."""
    t = table.detach().cpu()
    k, kp = eng.k, eng.kp
    if eng.internal_k == k:
        return t[:, :k].double(), bool((t[:, k:] == 0).all())
    d = torch.cat([t[:, :k], t[:, kp:kp + k]], 1).double()
    return d, bool((t[:, k:kp] == 0).all()) and bool((t[:, kp + k:] == 0).all())


def launched(run):
    """Names of the library's kernels that run() launched (torch.profiler, CUDA activities)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    return {e.key for e in prof.key_averages() if "kge_" in e.key}


def perturbed_term(model, ent, rel, triples, step, eta, factor, entities=None, max_lookups=32, device="cpu", **kw):
    """The sensitivity checks' perturbation: the gradient tables of one corruption alone, with its dL/dscore times
    `factor` (oracle_step with an external dL/dscore).  The corruption is the one whose replaced entity (one of
    `entities`, default any) has the fewest lookups in the step, at most max_lookups (None: any number), then the
    largest |dL/dscore|.  kw: oracle_step's rot_table / max_rel_size.  -> (corruption index, Step), or None where no
    corruption qualifies."""
    t = np.asarray(triples)
    corr = step.corr.cpu().numpy()
    lookups = np.bincount(np.concatenate([t[:, 0], t[:, 2], corr[:, 0], corr[:, 2]]), minlength=len(np.asarray(ent)))
    tiled = np.tile(t, (eta, 1))
    repl = np.where(corr[:, 0] != tiled[:, 0], corr[:, 0], corr[:, 2])
    keep = (corr[:, 0] == tiled[:, 0]).astype(np.uint8)
    g = step.dsn.abs().cpu().numpy()
    ok = g > 0
    if max_lookups is not None:
        ok &= lookups[repl] <= max_lookups
    if entities is not None:
        ok &= np.isin(repl, np.asarray(entities))
    cands = np.nonzero(ok)[0]
    if not len(cands):
        return None
    r = int(min(cands, key=lambda c: (lookups[repl[c]], -g[c])))
    i = r % len(t)
    one = oracle_step(model, ent, rel, t[i:i + 1], 1, [repl[r]], [keep[r]], dpos=[0.0],
                      dneg=[float(step.dsn[r]) * factor], device=device, **kw)
    return r, one


# --------------------------------------------------------------------------
# 1vsAll, KvsAll and relation prediction: a per-element bound
# --------------------------------------------------------------------------
OVA_C = 32  # the roundings of one term outside the chains: query vector, scale, exp, 1 / D, y, the chain pass's products


def abs_query(model, a, b):
    """On |tables|: the query of the slot whose two other rows are a and b, every product term counted positive, so
    that <abs_query, |x|> = abs_scores with x in that slot (HolE's scale included)."""
    if model == "DistMult":
        return a * b
    h = a.shape[1] // 2
    q = torch.cat([a[:, :h] * b[:, :h] + a[:, h:] * b[:, h:], a[:, :h] * b[:, h:] + a[:, h:] * b[:, :h]], 1)
    return q * (2.0 / h) if model == "HolE" else q


def row_stride(model, K):
    """The kernel's row stride ld for K internal columns: each half padded to a multiple of 4 floats."""
    halves = 1 if model in ("TransE", "DistMult") else 2
    return halves * (-(-(K // halves) // 4) * 4)


def ova_geometry(B, n_cand, relation=False):
    """(nsplit, xsplit) of a 1vsAll-family side: candidate ranges per query tile of the stats and dQ passes, and query-
    tile ranges per candidate tile of the dX pass (split on the relation side only)."""
    from ampligraph_b200.engine import one_vs_all_splits
    return one_vs_all_splits(B, n_cand), (one_vs_all_splits(n_cand, B) if relation else 1)


def ova_chains(B, n_cand, nsplit, xsplit, kvsall):
    """(n, n_loss): the longest fp32 chains one (query, candidate) term passes through on its way into a gradient
    element, and into the loss.  Gq: 32 fmas per candidate tile of the split, then the sum of nsplit partials; dX: 32
    per query tile of the split, then the sum of xsplit partials; D (1vsAll): two online updates (rescale and add, each
    with an expf) per tile of the split, four shuffle levels and the merge of nsplit partials."""
    n_qt, n_et = -(-B // 32), -(-n_cand // 32)
    per_split = -(-n_et // nsplit)
    n = max(32 * per_split + nsplit, 32 * -(-n_qt // xsplit) + xsplit)
    if kvsall:  # 4 elements per thread and tile, the warp sum
        return n, 4 * per_split + 5
    n_D = 10 * per_split + 6 * nsplit + 64
    return n + n_D, n_D


class OvaBound:
    """The per-element error bound of a 1vsAll-family step, side by side (add_side), checked with within_bound.

    A gradient element is a sum of terms g_be * d l_be / d theta, one per (query b, candidate e) pair of each side;
    |d l_be / d theta| <= d abs_score_be / d |theta| with abs_score_be = <abs_query_b, |x_e|>.  So for any weight W >= 0
    per pair, u * d/d|theta| sum W_be abs_score_be (u = 2^-24; autograd on |tables|, matmul form) bounds the element's
    error when W_be * u bounds the error of that pair's g_be relative to |d l_be / d theta|.  The weights:
      1vsAll, relation side: W = (|g| + P) (n + c) + P ((Lam_be + max_e Lam_be) / u + |lc - m| + 3 G)
      KvsAll:                W = |g| (n + c) + w (sig (1 - sig) Lam_be / u + c)
    P = lambda w_e p_be is the softmax part of g = P - lambda [e == t]; |g| (n + c) is the rounding of the chains the
    term passes through (ova_chains, plus the red.global.add chain into the row: n_red) and of c further operations;
    P (n + c) is p's relative rounding error (D's chain is part of n).  Lam_be = (ld + 4) u abs_score_be bounds the
    logit's error (ld fmas, the query's roundings, the scale), which moves p by at most p (Lam_be + max_e Lam_be)
    (p = exp(l_b) / sum exp(l_e) does not depend on m) and sigmoid by sig (1 - sig) Lam.  |lc - m| is the rounding of
    exp's argument, G = sum_e P_e (m - lc_e) that of the online rescales of D (m only grows, so their arguments
    telescope).  The multi-label rule's sig - y is an absolute error of c u (w: the reduction's weight).  Lam is 0 on
    dyadic tables, where every logit is exact.  A pair whose logit lies within Lam of +-75 may be clipped by one and not
    the other: it is charged in full ((|g| + P + lambda [e == t]) / u; KvsAll w |sig - y| / u).  A pair outside the clip
    range and not near it has g = 0 in both.  A1 (all W = 1) covers results below fp32's smallest normal.

    The loss: 1vsAll rows lambda (m + log D - l_t) with rounding (n_D + c) u (1 + |m| + |log D| + |l_t|) and logit
    error max Lam + Lam_t; KvsAll elements w (softplus(l) - y l) with rounding (n_loss + c) u (|softplus| + |y l|) and
    logit error Lam |sig - y|."""

    def __init__(self, model, ent, rel, triples, device="cpu"):
        self.model, self.device = model, torch.device(device)
        self.E = torch.as_tensor(np.asarray(ent), dtype=torch.float64, device=self.device)
        self.R = torch.as_tensor(np.asarray(rel), dtype=torch.float64, device=self.device)
        self.Ea = self.E.abs().requires_grad_(True)
        self.Ra = self.R.abs().requires_grad_(True)
        self.ld = row_stride(model, self.E.shape[1])
        self.A = [torch.zeros_like(self.E), torch.zeros_like(self.R)]
        self.A1 = [torch.zeros_like(self.E), torch.zeros_like(self.R)]
        self.loss = 0.0
        # red.global.add / in-place adds into one row: the chain pass per lookup on each side, and each side's dX add
        t = torch.as_tensor(np.asarray(triples), dtype=torch.long, device=self.device).reshape(-1, 3)
        lookups = max(int(torch.bincount(t[:, [0, 2]].reshape(-1)).max()) if len(t) else 0,
                      int(torch.bincount(t[:, 1]).max()) if len(t) else 0)
        self.n_red = 3 * lookups + 4

    def add_side(self, queries, side, reduction="sum", weight=1.0, labels=None, eps=0.0, nsplit=None, xsplit=None):
        """Adds one side: 's' / 'o' (1vsAll; KvsAll when `labels` is given) or 'p' (relation prediction, weight
        lambda).  nsplit / xsplit default to the kernel's (ova_geometry).  -> (nsplit, xsplit)."""
        import k_vs_all_oracle
        import one_vs_all_oracle
        import relation_prediction_oracle
        u, model, E, R, Ea, Ra = FP32_EPS, self.model, self.E, self.R, self.Ea, self.Ra
        t = torch.as_tensor(np.asarray(queries), dtype=torch.long, device=self.device).reshape(-1, 3)
        B = t.shape[0]
        s, p, o = t[:, 0], t[:, 1], t[:, 2]
        if side == "p":
            X, Xa, target = R, Ra, p
            q = relation_prediction_oracle.relation_query(model, E[s], E[o])
            qa = abs_query(model, Ea[s], Ea[o])
        else:
            X, Xa, target = E, Ea, (s if side == "s" else o)
            q = one_vs_all_oracle.query_vectors(model, side, E[s], R[p], E[o])
            qa = abs_query(model, *((Ra[p], Ea[o]) if side == "s" else (Ea[s], Ra[p])))
        n_cand = X.shape[0]
        geo = ova_geometry(B, n_cand, side == "p")
        nsplit, xsplit = nsplit or geo[0], xsplit or geo[1]
        n, n_loss = ova_chains(B, n_cand, nsplit, xsplit, labels is not None)
        n = n + self.n_red + OVA_C
        logits = (q @ X.T).detach()
        AS = qa @ Xa.T
        lam = (self.ld + 4) * u * AS.detach()
        inr = (logits.abs() <= ref_step.CLIP_HI).double()
        near = ((logits.abs() - ref_step.CLIP_HI).abs() < lam).double()
        lg = logits.clone().requires_grad_(True)
        if labels is None:
            loss = weight * one_vs_all_oracle.side_loss(lg, target, reduction).sum()
        else:
            y = k_vs_all_oracle.targets(labels, n_cand, eps, self.device)
            loss = k_vs_all_oracle.side_loss(lg, y, reduction).sum()
        g = torch.autograd.grad(loss, lg)[0].abs()
        if labels is None:
            lc, P, m, D = one_vs_all_oracle.side_softmax(logits, target, reduction)
            P = weight * P
            T = torch.zeros_like(P).scatter_(1, target[:, None], weight)
            G = (P * (m - lc)).sum(1, keepdim=True) / weight
            W = (inr * ((g + P) * n + P * ((lam + lam.max(1, keepdim=True).values) / u + (lc - m).abs() + 3 * G))
                 + near * (g + P + T) / u)
            lt = lc.gather(1, target[:, None])
            self.loss += weight * float(((n_loss + OVA_C) * u * (1 + m.abs() + torch.log(D).abs() + lt.abs())
                                         + lam.max(1, keepdim=True).values + lam.gather(1, target[:, None])).sum())
        else:
            w = 1.0 / n_cand if reduction == "mean" else 1.0
            lc = torch.clamp(logits, ref_step.CLIP_LO, ref_step.CLIP_HI)
            sig = torch.sigmoid(lc)
            W = inr * (g * n + w * (sig * (1 - sig) * lam / u + OVA_C)) + near * (g + w * (sig - y).abs()) / u
            sp = torch.nn.functional.softplus(lc)
            self.loss += w * float(((n_loss + OVA_C) * u * (sp + (y * lc).abs()) + lam * (sig - y).abs()).sum())
        for acc, wt in ((self.A, W), (self.A1, torch.ones_like(W))):
            Ea.grad = Ra.grad = None
            (wt * AS).sum().backward(retain_graph=True)
            acc[0] += Ea.grad
            acc[1] += Ra.grad
        return nsplit, xsplit

    def check(self, got_ent, got_rel, want_ent, want_rel, where=""):
        """Every element of both gradient tables within the bound (within_bound with the factors folded into A)."""
        for name, got, want, A, A1 in (("g_ent", got_ent, want_ent, self.A[0], self.A1[0]),
                                       ("g_rel", got_rel, want_rel, self.A[1], self.A1[1])):
            got = torch.as_tensor(np.asarray(got), dtype=torch.float64, device=self.device)
            want = torch.as_tensor(np.asarray(want), dtype=torch.float64, device=self.device)
            assert bool(torch.isfinite(got).all()), (where, name)
            ok, ratio = within_bound(got, want, A, A1, 1 - 8, 0)
            assert ok, (where, name, "worst error / bound %.3g" % ratio)

    def check_loss(self, got, want, where=""):
        """The loss within its bound (and within 1e-4 of its value, the looser check this one tightens)."""
        assert np.isfinite(got) and abs(got - want) <= min(self.loss, 1e-4 * abs(want)), (where, got, want, self.loss)
