"""RotatE's per-element bound (exact_oracle.RotatEBound) on the host: it is sound for an fp32 restatement of the
training kernels' arithmetic, sharp enough to reject that restatement with one defect, and the float64 oracle it is
measured against is the reference's gradient.

The restatement follows the rot_* functions of kge_train_common.cuh and kge_train_rot_kernel's order of operations in
numpy float32 (fmaf through float64); its sqrt / rsqrt are the correctly rounded values pushed by the MUFU error bound
(EPS_SQRT / EPS_RSQ) to one side, both sides tried."""
import numpy as np
import pytest
import torch

import exact_oracle as xo
from oracle import ref_step

F = np.float32
TINY = F(2.0 ** -126)


def fma(a, b, c):
    return (np.float64(a) * np.float64(b) + np.float64(c)).astype(F)


class Restatement:
    """One KGE_STEP_BACKWARD_EXT step in fp32 -> (sp, sn, g_ent, g_rel).  mutant: None or (kind, corruption index)."""

    def __init__(self, push=1.0, mutant=None):
        self.push, self.mutant = push, mutant

    def sqrt(self, x):
        return F(np.sqrt(np.float64(x)) * (1 + self.push * xo.EPS_SQRT))

    def rsqrt(self, x):
        return F((1.0 / np.sqrt(np.float64(np.maximum(x, TINY)))) * (1 + self.push * xo.EPS_RSQ))

    def modsum(self, re, im):
        return F(np.sum(self.sqrt(fma(im, im, re * re)), dtype=F))

    def unit(self, re, im, g):
        inv = F(g) * self.rsqrt(fma(im, im, re * re))
        return re * inv, im * inv

    @staticmethod
    def rotate(xr, xi, c, s):
        return fma(-xi, s, xr * c), fma(xr, s, xi * c)

    def back(self, a, b, c, s, j):
        if self.mutant == ("cos_for_sin", j):
            s = c
        return fma(-b, s, -a * c), fma(-b, c, a * s)

    def run(self, ent, rel, triples, ne, nk, eta, dpos, dneg, max_rel_size=None):
        ent, rel = np.asarray(ent, F), np.asarray(rel, F)
        K = ent.shape[1]
        h = K // 2
        div, inv_div = xo.rotation_divisor32(K, max_rel_size or rel.shape[0])
        ct, st = xo.rotation_table(rel[:, :h], div)
        B = len(triples)
        ne, nk = np.asarray(ne).reshape(eta, B), np.asarray(nk).reshape(eta, B)
        g_ent, g_rel = np.zeros_like(ent), np.zeros_like(rel)
        sp, sn = np.zeros(B, F), np.zeros((eta, B), F)
        mut = self.mutant or (None, -1)

        def add(row, cols, v, j):
            reps = 2 if mut == ("double", j) else 0 if mut == ("drop", j) else 1
            for _ in range(reps):
                g_ent[row, cols] = g_ent[row, cols] + v

        for i, (s, p, o) in enumerate(triples):
            c, sg = ct[p], st[p]
            xr, xi, orr, oi = ent[s, :h], ent[s, h:], ent[o, :h], ent[o, h:]
            Yr, Yi = self.rotate(xr, xi, c, sg)
            sp[i] = -self.modsum(Yr - orr, Yi - oi)
            Zor, Zoi, Zsr, Zsi, Aphi = (np.zeros(h, F) for _ in range(5))
            for j in sorted(range(eta), key=lambda j: nk[j, i]):  # the kernel's slots: subject-replaced first
                r, side, g = ne[j, i], int(nk[j, i]), F(dneg[j * B + i])
                if mut == ("flip", j * B + i):
                    side ^= 1
                rr, ri = ent[r, :h], ent[r, h:]
                if side == 0:  # subject replaced: R(phi) r - o
                    sn[j, i] = -self.modsum(fma(-ri, sg, fma(rr, c, -orr)), fma(ri, c, fma(rr, sg, -oi)))
                    yr, yi = self.rotate(rr, ri, c, sg)
                    a, b = self.unit(yr - orr, yi - oi, g)
                    if mut == ("drop", j * B + i):
                        continue
                    Zsr, Zsi = Zsr + a, Zsi + b
                    Aphi = fma(-b, yr, fma(a, yi, Aphi))
                    br, bi = self.back(a, b, c, sg, j * B + i)
                    add(r, slice(0, h), br, j * B + i)
                    add(r, slice(h, K), bi, j * B + i)
                else:  # object replaced: y(s) - r
                    sn[j, i] = -self.modsum(Yr - rr, Yi - ri)
                    a, b = self.unit(Yr - rr, Yi - ri, g)
                    if mut == ("drop", j * B + i):
                        continue
                    Zor, Zoi = Zor + a, Zoi + b
                    if mut == ("swap", j * B + i):
                        a, b = b, a
                    add(r, slice(0, h), a, j * B + i)
                    add(r, slice(h, K), b, j * B + i)
            a, b = self.unit(Yr - orr, Yi - oi, F(dpos[i]))
            Zr, Zi = a + Zor, b + Zoi
            br, bi = self.back(Zr, Zi, c, sg, -1)
            g_ent[s, :h] += br
            g_ent[s, h:] += bi
            g_ent[o, :h] += a + Zsr
            g_ent[o, h:] += b + Zsi
            dphi = fma(-Zi, Yr, fma(Zr, Yi, Aphi))
            g_rel[p, :h] += dphi if mut == ("no_inv_div", -1) else F(inv_div) * dphi
        return sp, sn.reshape(-1), g_ent, g_rel


def _case(seed, k=8, E=12, R=3, B=4, eta=5, scale=1.0):
    rng = np.random.default_rng(seed)
    K = 2 * k
    ent = (rng.uniform(-1, 1, (E, K)) * scale).astype(F)
    rel = rng.uniform(-1, 1, (R, K)).astype(F)
    t = np.stack([rng.integers(0, E, B), rng.integers(0, R, B), rng.integers(0, E, B)], 1).astype(np.int32)
    ne = rng.integers(0, E, eta * B).astype(np.int32)
    nk = rng.integers(0, 2, eta * B).astype(np.uint8)
    dpos = rng.uniform(-1, 1, B).astype(F)
    dneg = rng.uniform(-1, 1, eta * B).astype(F)
    return ent, rel, t, ne, nk, eta, dpos, dneg


def _check(case, out, step=None):
    ent, rel, t, ne, nk, eta, dpos, dneg = case
    if step is None:
        step = xo.oracle_step("RotatE", ent, rel, t, eta, ne, nk, dpos=dpos, dneg=dneg, rot_table=True)
    bound = xo.RotatEBound(ent, rel, t, step, eta)
    sp, sn, ge, gr = out
    res = bound.check(ge, gr, step.g_ent, step.g_rel)
    res.append(("sp",) + bound.check_scores(sp, step.sp, "sp"))
    res.append(("sn",) + bound.check_scores(sn, step.sn, "sn"))
    return res, step, bound


@pytest.mark.parametrize("push", [1.0, -1.0])
@pytest.mark.parametrize("seed,scale", [(0, 1.0), (1, 1.0), (2, 2.0 ** -56), (3, 2.0 ** 40)])
def test_bound_is_sound(seed, scale, push):
    """The restatement stays within the bound, sqrt / rsqrt pushed to either side, at unit scale, at rows of 2^-56
    (|v|^2 in [2^-126, 1e-30)) and at 2^40."""
    case = _case(seed, scale=scale)
    res, _, _ = _check(case, Restatement(push).run(*case))
    assert all(ok for _, ok, _ in res), res


def test_bound_is_sound_near_zero_residual():
    """o = R(phi) s up to an ulp: the positive's residual is ~1e-8 and its unit vector ill-conditioned."""
    case = list(_case(4))
    ent, rel, t = case[0].copy(), case[1], case[2]
    h = ent.shape[1] // 2
    div, _ = xo.rotation_divisor32(ent.shape[1], rel.shape[0])
    c, s = xo.rotation_table(rel[t[0, 1], :h], div)
    yr, yi = Restatement.rotate(ent[t[0, 0], :h], ent[t[0, 0], h:], c, s)
    ent[t[0, 2], :h], ent[t[0, 2], h:] = np.nextafter(yr, F(2)), yi
    case[0] = ent
    for push in (1.0, -1.0):
        res, step, _ = _check(case, Restatement(push).run(*case))
        assert all(ok for _, ok, _ in res), res
    assert float(-step.sp[0]) < 1e-6


MUTANTS = ["drop", "double", "flip", "swap", "cos_for_sin", "no_inv_div"]


@pytest.mark.parametrize("kind", MUTANTS)
def test_bound_rejects_mutants(kind):
    """Each defect of the restatement fails the check: one term dropped (every corruption with a term above 2^-10 of
    its element's A, in turn), doubled, its side flipped, its re / im halves swapped or cos used for sin in its
    back-rotation; inv_div omitted from the relation gradient."""
    case = _case(7)
    ent, rel, t, ne, nk, eta, dpos, dneg = case
    res, step, bound = _check(case, Restatement().run(*case))
    assert all(ok for _, ok, _ in res), res
    B = len(t)
    if kind == "no_inv_div":
        targets = [-1]
    elif kind == "swap":
        targets = [r for r in range(eta * B) if nk[r] == 1]
    elif kind == "cos_for_sin":
        targets = [r for r in range(eta * B) if nk[r] == 0]
    else:
        targets = list(range(eta * B))
    for r in targets:
        if kind == "drop":  # the term: one corruption's gradient alone
            j, i = divmod(r, B)
            one = xo.oracle_step("RotatE", ent, rel, t[i:i + 1], 1, ne[r:r + 1], nk[r:r + 1], dpos=[0.0],
                                 dneg=dneg[r:r + 1], rot_table=True, max_rel_size=rel.shape[0])
            big = (one.g_ent.abs() > 2.0 ** -10 * bound.A[0]).any() or (one.g_rel.abs() > 2.0 ** -10 * bound.A[1]).any()
            if not bool(big):
                continue
        out = Restatement(mutant=(kind, r)).run(*case)
        res, _, _ = _check(case, out, step)
        assert not all(ok for name, ok, _ in res if name.startswith("g_")), (kind, r, res)


@pytest.mark.parametrize("rot_table", [False, True])
def test_oracle_matches_reference_autograd(rot_table):
    """oracle_step's float64 RotatE gradient is ref_step.compute_scores under autograd (the reference's), and with
    the kernels' rotation table it differs from it only by the table's fp32 rounding."""
    ent, rel, t, ne, nk, eta, dpos, dneg = _case(9)
    step = xo.oracle_step("RotatE", ent, rel, t, eta, ne, nk, dpos=dpos, dneg=dneg, rot_table=rot_table)
    E = torch.tensor(ent, dtype=torch.float64, requires_grad=True)
    R = torch.tensor(rel, dtype=torch.float64, requires_grad=True)
    tt = torch.as_tensor(t, dtype=torch.long)
    corr = ref_step.corrupt(tt, eta, torch.as_tensor(nk, dtype=torch.long), torch.as_tensor(ne, dtype=torch.long))
    sp = ref_step.compute_scores("RotatE", E[tt[:, 0]], R[tt[:, 1]], E[tt[:, 2]], rel.shape[0])
    sn = ref_step.compute_scores("RotatE", E[corr[:, 0]], R[corr[:, 1]], E[corr[:, 2]], rel.shape[0])
    ((sp * torch.as_tensor(dpos, dtype=torch.float64)).sum() + (sn * torch.as_tensor(dneg, dtype=torch.float64)).sum()).backward()
    tol = 2.0 ** -40 if not rot_table else 2.0 ** -18
    for got, want in ((step.g_ent, E.grad), (step.g_rel, R.grad)):
        assert float((got - want).abs().max()) <= tol * float(want.abs().max())


def test_oracle_matches_central_differences():
    """The float64 oracle's gradient against central differences of its own objective, every element."""
    ent, rel, t, ne, nk, eta, dpos, dneg = _case(10, k=3, E=6, R=2, B=2, eta=3)
    step = xo.oracle_step("RotatE", ent, rel, t, eta, ne, nk, dpos=dpos, dneg=dneg)
    tt = torch.as_tensor(t, dtype=torch.long)
    corr = ref_step.corrupt(tt, eta, torch.as_tensor(nk, dtype=torch.long), torch.as_tensor(ne, dtype=torch.long))

    def f(E, R):
        sp = xo.scores("RotatE", E[tt[:, 0]], R[tt[:, 1]], E[tt[:, 2]], R.shape[0])
        sn = xo.scores("RotatE", E[corr[:, 0]], R[corr[:, 1]], E[corr[:, 2]], R.shape[0])
        return float((sp * torch.as_tensor(dpos, dtype=torch.float64)).sum()
                     + (sn * torch.as_tensor(dneg, dtype=torch.float64)).sum())

    E0, R0 = torch.tensor(ent, dtype=torch.float64), torch.tensor(rel, dtype=torch.float64)
    eps = 1e-6
    for which, X, G in (("ent", E0, step.g_ent), ("rel", R0, step.g_rel)):
        for idx in np.ndindex(*X.shape):
            Xp, Xm = X.clone(), X.clone()
            Xp[idx] += eps
            Xm[idx] -= eps
            fd = (f(Xp, R0) - f(Xm, R0)) / (2 * eps) if which == "ent" else (f(E0, Xp) - f(E0, Xm)) / (2 * eps)
            assert abs(fd - float(G[idx])) <= 1e-6 * (1 + abs(fd)), (which, idx, fd, float(G[idx]))


def test_fused_loss_bound_covers_score_errors():
    """self_adversarial: the Hessian term moves dL/dscore by at most |H| ds; pushing every score of the float64 oracle
    by its bound moves g by no more than RotatEBound's dg allows (the bound's use of the Hessian is first order)."""
    ent, rel, t, ne, nk, eta, _, _ = _case(11)
    lp = {"margin": 3.0, "alpha": 0.5}
    step = xo.oracle_step("RotatE", ent, rel, t, eta, ne, nk, loss="self_adversarial", loss_params=lp, rot_table=True)
    bound = xo.RotatEBound(ent, rel, t, step, eta, loss="self_adversarial", loss_params=lp)
    B = len(t)
    sp, sn = step.sp.clone(), step.sn.reshape(eta, B).clone()
    ds_p, ds_n = bound.score_err[:B], bound.score_err[B:].reshape(eta, B)
    hp, hn = xo.loss_score_sensitivity("self_adversarial", lp, sp, sn, ds_p, ds_n)
    for sgn in (1.0, -1.0):
        s = torch.cat([(sp + sgn * ds_p)[None], sn - sgn * ds_n], 0).requires_grad_(True)
        L = ref_step.per_positive_loss("self_adversarial", s[0], s[1:], margin=3.0, alpha=0.5).sum()
        g = torch.autograd.grad(L, s)[0]
        assert bool(((g[0] - step.dsp).abs() <= 1.01 * hp + 1e-300).all())
        assert bool(((g[1:] - step.dsn.reshape(eta, B)).abs() <= 1.01 * hn + 1e-300).all())
