"""The per-element bound of DistMult, ComplEx, HolE and TransE training (exact_oracle.TrilinearBound) on the host: it is
sound for an fp32 evaluation of the same step, and sharp enough to reject that evaluation with one defect that the
suite's older check, test_gpu_parity._close at rtol 1e-4 of the table's largest element, accepts.

The fp32 evaluation is oracle_step(..., dtype=torch.float32): the reference's graph under autograd in fp32, a legitimate
evaluation of the step in another order of operations than the kernels'.  The tables are Glorot-scaled
(uniform +-sqrt(6 / (rows + K))) and k = 100 is not a power of two, so HolE's 2 / k is inexact."""
import numpy as np
import pytest
import torch

import exact_oracle as xo
from test_gpu_parity import _close

MODELS = ["DistMult", "ComplEx", "HolE", "TransE"]
LOSSES = [("nll", {}), ("multiclass_nll", {}), ("self_adversarial", {"margin": 3.0, "alpha": 0.5}),
          ("pairwise", {"margin": 0.5}), ("absolute_margin", {"margin": 1.0}), ("ext", {})]
LOSS_IDS = [l for l, _ in LOSSES]


def glorot(rng, rows, K):
    lim = np.sqrt(6.0 / (rows + K))
    return rng.uniform(-lim, lim, (rows, K)).astype(np.float32)


def case(model, eta, seed, k=100, E=200, R=7, B=40):
    """Glorot tables, Zipf positives, uniform corruptions of which a few replace an entity with itself (N = P)."""
    rng = np.random.default_rng(seed)
    K = xo.internal_k(model, k)
    ent, rel = glorot(rng, E, K), glorot(rng, R, K)
    t = xo.zipf_triples(E, R, B, rng)
    ne = rng.integers(0, E, eta * B).astype(np.int32)
    nk = rng.integers(0, 2, eta * B).astype(np.uint8)
    tiled = np.tile(t, (eta, 1))
    same = rng.random(eta * B) < 0.03
    ne[same] = np.where(nk[same] == 1, tiled[same, 2], tiled[same, 0])
    ext = dict(dpos=rng.uniform(-1, 1, B).astype(np.float32), dneg=rng.uniform(-1, 1, eta * B).astype(np.float32))
    return ent, rel, t, ne, nk, ext


def steps(model, loss, lp, reduction, eta, seed=0, **shape):
    ent, rel, t, ne, nk, ext = case(model, eta, seed, **shape)
    lp = dict(lp, reduction=reduction)
    kw = dict(ext) if loss == "ext" else dict(loss=loss, loss_params=lp)
    ref = xo.oracle_step(model, ent, rel, t, eta, ne, nk, **kw)
    f32 = xo.oracle_step(model, ent, rel, t, eta, ne, nk, dtype=torch.float32, **kw)
    bound = xo.TrilinearBound(model, ent, rel, t, ref, eta, loss=None if loss == "ext" else loss, loss_params=lp)
    return (ent, rel, t, ne, nk), ref, f32, bound


def one_term(model, data, r, g):
    """The gradient tables of corruption r alone with dL/dscore g (the term it adds to its rows)."""
    ent, rel, t, ne, nk = data
    i = r % len(t)
    return xo.oracle_step(model, ent, rel, t[i:i + 1], 1, ne[r:r + 1], nk[r:r + 1], dpos=[0.0], dneg=[g])


def replaced_terms(model, data, ref):
    """Per corruption, the largest element of the term it adds to its replaced row (float64)."""
    ent, rel, t, ne, nk = data
    E, R = torch.as_tensor(ent, dtype=torch.float64), torch.as_tensor(rel, dtype=torch.float64)
    c = ref.corr
    S, O = E[c[:, 0]].clone().requires_grad_(True), E[c[:, 2]].clone().requires_grad_(True)
    (xo.scores(model, S, R[c[:, 1]], O) * ref.dsn).sum().backward()
    return torch.where(torch.as_tensor(nk, dtype=torch.bool)[:, None], O.grad, S.grad).abs().max(1).values.numpy()


def sensitive_corruption(model, data, ref, cap):
    """A corruption whose replaced entity has at most 32 lookups in the step and whose term stays below cap: the fewest
    lookups, then the largest term."""
    ent, rel, t, ne, nk = data
    corr = ref.corr.numpy()
    lookups = np.bincount(np.concatenate([t[:, 0], t[:, 2], corr[:, 0], corr[:, 2]]), minlength=len(ent))
    term = replaced_terms(model, data, ref)
    cand = [r for r in range(len(ne)) if lookups[ne[r]] <= 32 and 0 < term[r] < cap]
    assert cand, "no corruption with a replaced entity of at most 32 lookups and a term below the cap"
    return min(cand, key=lambda r: (lookups[ne[r]], -term[r]))


@pytest.mark.parametrize("eta", [10, 33])
@pytest.mark.parametrize("reduction", ["sum", "mean"])
@pytest.mark.parametrize("loss,lp", LOSSES, ids=LOSS_IDS)
@pytest.mark.parametrize("model", MODELS)
def test_bound_is_sound(model, loss, lp, reduction, eta):
    """The fp32 evaluation lies within the bound: scores, loss and every gradient element (eta = 10, and 33 > 32:
    self_adversarial's looped branch; mean with eta not a power of two: w = 1 / eta inexact)."""
    if loss == "ext" and reduction == "mean":
        pytest.skip("an external dL/dscore has no reduction")
    _, ref, f32, bound = steps(model, loss, lp, reduction, eta)
    res = bound.check(f32.g_ent, f32.g_rel, ref.g_ent, ref.g_rel)
    res.append(("sp",) + bound.check_scores(f32.sp, ref.sp, "sp"))
    res.append(("sn",) + bound.check_scores(f32.sn, ref.sn, "sn"))
    assert all(ok for _, ok, _ in res), res
    if loss != "ext":
        assert abs(f32.loss - ref.loss) <= bound.loss_err, (f32.loss, ref.loss, bound.loss_err)


@pytest.mark.parametrize("loss,lp", LOSSES[:3] + LOSSES[5:], ids=LOSS_IDS[:3] + LOSS_IDS[5:])
@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("defect", ["perturbed", "dropped"])
def test_bound_rejects_one_defect(defect, model, loss, lp):
    """The fp32 evaluation with one corruption's dL/dscore multiplied by 1 + 2^-10, or with its term removed, fails
    the bound.  _close (rtol 1e-4 of the largest element) accepts the perturbed one: at 1,500 Zipf positives over 2,000
    entities the hot rows set the largest element, as on the workloads' shapes.  It accepts a dropped term only when the
    term is below its tolerance: with an external dL/dscore (uniform in [-1, 1], so some are small) the dropped term is
    one below half of it, and _close accepts it; a fused loss's terms here all exceed it."""
    data, ref, f32, bound = steps(model, loss, lp, "sum", 10, E=2000, B=1500)
    small = defect == "dropped" and loss == "ext"
    cap = 0.5e-4 * float(ref.g_ent.abs().max()) if small else np.inf
    r = sensitive_corruption(model, data, ref, cap)
    g = float(ref.dsn[r]) * (2.0 ** -10 if defect == "perturbed" else -1.0)
    one = one_term(model, data, r, g)
    got_e, got_r = f32.g_ent.double() + one.g_ent, f32.g_rel.double() + one.g_rel
    assert not all(ok for _, ok, _ in bound.check(got_e, got_r, ref.g_ent, ref.g_rel)), (defect, r)
    if defect == "perturbed" or small:
        assert _close(got_e.numpy(), ref.g_ent.numpy()) and _close(got_r.numpy(), ref.g_rel.numpy())


def test_fused_loss_bound_covers_score_errors():
    """multiclass_nll on ComplEx: pushing every score of the float64 oracle by its bound moves dL/dscore by no more than
    the first-order Hessian term of loss_error (the bound's use of the Hessian is first order)."""
    data, ref, _, bound = steps("ComplEx", "multiclass_nll", {}, "sum", 10)
    B, eta = len(data[2]), 10
    sp, sn = ref.sp.clone(), ref.sn.reshape(eta, B).clone()
    ds_p, ds_n = bound.score_err[:B], bound.score_err[B:].reshape(eta, B)
    hp, hn = xo.loss_score_sensitivity("multiclass_nll", {}, sp, sn, ds_p, ds_n)
    from oracle import ref_step
    for sgn in (1.0, -1.0):
        s = torch.cat([(sp + sgn * ds_p)[None], sn - sgn * ds_n], 0).requires_grad_(True)
        L = ref_step.per_positive_loss("multiclass_nll", s[0], s[1:]).sum()
        g = torch.autograd.grad(L, s)[0]
        assert bool(((g[0] - ref.dsp).abs() <= 1.01 * hp + 1e-300).all())
        assert bool(((g[1:] - ref.dsn.reshape(eta, B)).abs() <= 1.01 * hn + 1e-300).all())


def test_transe_premise_is_asserted():
    """A TransE residual of exactly 0 (o = s + p on a grid) violates the premise: the bound refuses the data."""
    rng = np.random.default_rng(1)
    ent, rel = xo.grid_table(rng, 6, 8), xo.grid_table(rng, 2, 8)
    ent[1] = ent[0] + rel[0]
    t = np.array([[0, 0, 1]], np.int32)
    ref = xo.oracle_step("TransE", ent, rel, t, 1, [2], [1], dpos=[1.0], dneg=[1.0])
    with pytest.raises(AssertionError, match="premise"):
        xo.TrilinearBound("TransE", ent, rel, t, ref, 1)
