"""The float64 training-step oracle (tests/exact_oracle.py) on the host: its edge rules, the exactness claim the GPU
tests stand on (fp32 evaluation of a step on dyadic tables equals float64, in two summation orders), and how much the
table-wide tolerance of the other training tests can hide."""
import numpy as np
import pytest
import torch

import exact_oracle as xo
from oracle import ref_step


def _one(loss, P, N, **lp):
    """dL/dP, dL/dN of one positive with one corruption (float64 autograd)."""
    sp = torch.tensor([P], dtype=torch.float64, requires_grad=True)
    sn = torch.tensor([[N]], dtype=torch.float64, requires_grad=True)
    ref_step.per_positive_loss(loss, sp, sn, **lp).sum().backward()
    return float(sp.grad[0]), float(sn.grad[0, 0])


@pytest.mark.parametrize("loss", ["nll", "multiclass_nll"])
def test_clip_passes_gradient_at_the_bound_and_not_beyond(loss):
    step = 2.0 ** -4
    for bound in (-75.0, 75.0):
        beyond = bound + (step if bound > 0 else -step)
        # (the partner score sits at the bound too, so that multiclass_nll's softmax is not saturated)
        dP, dN = _one(loss, bound, bound)
        assert dP != 0.0 and dN != 0.0, (loss, bound)
        dP, _ = _one(loss, beyond, bound)
        assert dP == 0.0, (loss, beyond)
        _, dN = _one(loss, bound, beyond)
        assert dN == 0.0, (loss, beyond)


def test_hinge_tie_passes_gradient():
    # pairwise: margin - P + N = 0; absolute_margin: margin + N = 0 (TF maximum() gives the tie to its first argument)
    dP, dN = _one("pairwise", 0.5, -0.5, margin=1.0)
    assert (dP, dN) == (-1.0, 1.0)
    dP, dN = _one("pairwise", 0.5, -0.5 - 2.0 ** -4, margin=1.0)
    assert (dP, dN) == (0.0, 0.0)
    _, dN = _one("absolute_margin", 0.5, -1.0, margin=1.0)
    assert dN == 1.0
    _, dN = _one("absolute_margin", 0.5, -1.0 - 2.0 ** -4, margin=1.0)
    assert dN == 0.0


def test_abs_gradient_at_zero_is_zero():
    e = torch.tensor([[0.5, 1.0]], dtype=torch.float64, requires_grad=True)
    p = torch.tensor([[0.5, -0.5]], dtype=torch.float64, requires_grad=True)
    o = torch.tensor([[1.0, 1.0]], dtype=torch.float64, requires_grad=True)
    xo.scores("TransE", e, p, o).sum().backward()  # residual (0, -0.5)
    assert e.grad.tolist() == [[0.0, 1.0]] and o.grad.tolist() == [[0.0, -1.0]]


def test_rotate_zero_modulus_gradient_is_zero_where_the_reference_is_nan():
    s = torch.tensor([[0.5, -0.25, 0.75, 1.0]], dtype=torch.float64)
    o = s.clone()
    o[0, 1] += 0.5  # complex column 1 differs, column 0 is an exactly zero residual
    p = torch.zeros((1, 4), dtype=torch.float64)  # theta = 0
    grads = []
    for fn in (xo.scores, ref_step.compute_scores):
        ss, pp, oo = (x.clone().requires_grad_(True) for x in (s, p, o))
        fn("RotatE", ss, pp, oo, 1).sum().backward()
        grads.append(ss.grad)
    ours, theirs = grads
    assert bool(torch.isfinite(ours).all()) and ours[0, 0] == 0 and ours[0, 2] == 0 and ours[0, 1] != 0
    assert bool(torch.isnan(theirs[0, [0, 2]]).all())  # the reference's sqrt gradient at 0
    assert torch.equal(ours[0, [1, 3]], theirs[0, [1, 3]])


def test_assert_fp32_exact():
    xo.assert_fp32_exact(torch.tensor([1.0, 2.0 ** -30, 3.0 * 2.0 ** 20], dtype=torch.float64))
    with pytest.raises(AssertionError):
        xo.assert_fp32_exact(torch.tensor([1.0 + 2.0 ** -30], dtype=torch.float64))


# ---------------------------------------------------------------------------
# the exactness claim
# ---------------------------------------------------------------------------
def _reversed_columns(model, K):
    """A column permutation that reverses the summation order within each half of a row (the halves stay put)."""
    if model in ("DistMult", "TransE"):
        return np.arange(K)[::-1].copy()
    h = K // 2
    return np.concatenate([np.arange(h)[::-1], h + np.arange(h)[::-1]])


# (model, k, eta, E, R, B, negatives): the shapes of tests/test_gpu_exact_training.py's exact-equality tests
SHAPES = [("DistMult", 16, 8, 400, 7, 600, "uniform"), ("DistMult", 400, 8, 400, 7, 600, "uniform"),
          ("ComplEx", 16, 8, 400, 7, 600, "uniform"), ("ComplEx", 200, 8, 400, 7, 600, "uniform"),
          ("HolE", 8, 8, 400, 7, 600, "uniform"), ("HolE", 128, 8, 400, 7, 600, "uniform"),
          ("TransE", 16, 8, 400, 7, 600, "uniform"), ("TransE", 200, 8, 400, 7, 600, "uniform"),
          ("DistMult", 1100, 7, 300, 5, 200, "uniform"), ("ComplEx", 520, 7, 300, 5, 200, "uniform"),
          ("HolE", 1024, 7, 300, 5, 200, "uniform"), ("TransE", 600, 7, 300, 5, 200, "uniform"),
          ("DistMult", 400, 20, 3000, 9, 2000, "uniform"), ("ComplEx", 200, 10, 700, 9, 4000, "skewed"),
          ("DistMult", 8, 5, 100000, 9, 20000, "uniform"), ("HolE", 128, 4, 400, 9, 700, "uniform")]


# pairwise with reduction mean is dyadic only for eta a power of two
EXACT_CASES = [pytest.param(*shape, kind, id="%s-%d-%d-%s-%s" % (shape[0], shape[1], shape[2], shape[6], kind))
               for shape in SHAPES
               for kind in ["pairwise", "absolute_margin", "ext"] + (["pairwise_mean"] if shape[2] & (shape[2] - 1) == 0 else [])]


@pytest.mark.parametrize("model,k,eta,E,R,B,negs,kind", EXACT_CASES)
def test_fp32_step_is_exact_on_the_grid(model, k, eta, E, R, B, negs, kind):
    """The fp32 evaluation of the step equals the float64 one bit for bit, in the natural order and with the positives
    permuted and every row's columns reversed (other summation orders of the scores and of the gradient rows)."""
    rng = np.random.default_rng(k * 1000 + eta)
    K = xo.internal_k(model, k)
    ent, rel = xo.grid_table(rng, E, K), xo.grid_table(rng, R, K)
    t = xo.zipf_triples(E, R, B, rng)
    if negs == "skewed":
        ne = rng.choice(np.array([3, 77, 500], np.int32), B * eta)
    else:
        ne = rng.integers(0, E, B * eta).astype(np.int32)
    nk = rng.integers(0, 2, B * eta).astype(np.uint8)
    loss = "absolute_margin" if kind == "absolute_margin" else "pairwise"
    lp = {"margin": 0.5, "reduction": "mean"} if kind == "pairwise_mean" else {"margin": 1.0}
    ext = {}
    if kind == "ext":
        vals = np.array([-1.0, -0.5, 0.0, 0.5, 1.0])
        ext = dict(dpos=rng.choice(vals, B), dneg=rng.choice(vals, eta * B))
    ref = xo.oracle_step(model, ent, rel, t, eta, ne, nk, loss=loss, loss_params=lp, **ext)
    for x in (ref.sp, ref.sn, ref.g_ent, ref.g_rel):
        xo.assert_fp32_exact(x)
    f32 = xo.oracle_step(model, ent, rel, t, eta, ne, nk, loss=loss, loss_params=lp, dtype=torch.float32, **ext)
    # the other order: positives permuted (so are their corruptions), columns reversed within each half
    perm, cols = rng.permutation(B), _reversed_columns(model, K)
    ext2 = {}
    if ext:
        ext2 = dict(dpos=ext["dpos"][perm], dneg=ext["dneg"].reshape(eta, B)[:, perm].reshape(-1))
    f32b = xo.oracle_step(model, ent[:, cols], rel[:, cols], t[perm], eta, ne.reshape(eta, B)[:, perm].reshape(-1),
                          nk.reshape(eta, B)[:, perm].reshape(-1), loss=loss, loss_params=lp, dtype=torch.float32, **ext2)
    inv = np.argsort(perm)
    back = dict(sp=f32b.sp[inv], sn=f32b.sn.reshape(eta, B)[:, inv].reshape(-1),
                g_ent=f32b.g_ent[:, np.argsort(cols)], g_rel=f32b.g_rel[:, np.argsort(cols)])
    for name in ("sp", "sn", "g_ent", "g_rel"):
        want = getattr(ref, name)
        assert torch.equal(getattr(f32, name).double(), want), name
        assert torch.equal(back[name].double(), want), name + " (other order)"
    if ref.loss is not None:
        assert f32.loss == ref.loss


def test_fp32_step_is_exact_cfg2_shape():
    """bench.py's shape (ComplEx k=200, eta=10, 14,505 entities, 27,212 Zipf positives) on the 5-point grid."""
    rng = np.random.default_rng(2)
    E, R, B, eta, K = 14505, 237, 27212, 10, 400
    ent, rel = xo.grid_table(rng, E, K), xo.grid_table(rng, R, K)
    t = xo.zipf_triples(E, R, B, rng)
    ne, nk = rng.integers(0, E, B * eta).astype(np.int32), rng.integers(0, 2, B * eta).astype(np.uint8)
    ref = xo.oracle_step("ComplEx", ent, rel, t, eta, ne, nk, loss="pairwise", loss_params={"margin": 1.0}, chunk=4096)
    f32 = xo.oracle_step("ComplEx", ent, rel, t, eta, ne, nk, loss="pairwise", loss_params={"margin": 1.0}, chunk=2048,
                         dtype=torch.float32)
    for name in ("sp", "sn", "g_ent", "g_rel"):
        xo.assert_fp32_exact(getattr(ref, name), name)
        assert torch.equal(getattr(f32, name).double(), getattr(ref, name)), name
    assert f32.loss == ref.loss


# ---------------------------------------------------------------------------
# what a table-wide tolerance can hide
# ---------------------------------------------------------------------------
def cold_rows_cfg2(rtol=1e-4):
    """cfg2's step as tests/test_gpu_parity.py draws it (ComplEx k=200, eta=10, 14,505 entities, 27,212 Zipf positives,
    Glorot-uniform tables, uniform injected corruptions, self_adversarial): (entity rows with a gradient, those among
    them whose largest |g| is below rtol times the table's largest |G|, the coldest row's largest |g| over |G|)."""
    rng = np.random.default_rng(101)
    E, R, k, eta, B = 14505, 237, 200, 10, 27212
    K = 2 * k
    ent = rng.uniform(-np.sqrt(6.0 / (E + K)), np.sqrt(6.0 / (E + K)), (E, K)).astype(np.float32)
    rel = rng.uniform(-np.sqrt(6.0 / (R + K)), np.sqrt(6.0 / (R + K)), (R, K)).astype(np.float32)
    t = xo.zipf_triples(E, R, B, rng)
    ne, nk = rng.integers(0, E, B * eta).astype(np.int32), rng.integers(0, 2, B * eta).astype(np.uint8)
    ref = xo.oracle_step("ComplEx", ent, rel, t, eta, ne, nk, loss="self_adversarial",
                         loss_params={"margin": 3.0, "alpha": 0.5}, chunk=4096)
    row_max = ref.g_ent.abs().max(1).values
    touched = row_max > 0
    G = float(row_max.max())
    cold = touched & (row_max < rtol * G)
    return int(touched.sum()), int(cold.sum()), float(row_max[touched].min()) / G


def test_table_wide_tolerance_at_cfg2():
    """How much the 1e-4-of-the-table's-maximum comparison of the other training tests can hide at cfg2's shape: no
    entity row falls below it (every row is hit; the coldest row's largest entry is about 1 % of the table's), so a
    whole cold row cannot vanish unnoticed there.  The exact tests need no such argument."""
    touched, cold, coldest = cold_rows_cfg2()
    print("cfg2: %d of %d entity rows with a gradient have max|g| < 1e-4 max|G|; coldest row %.3g of max|G|"
          % (cold, touched, coldest))
    assert touched == 14505 and cold == 0 and 1e-3 < coldest < 0.1
