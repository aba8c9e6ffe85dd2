"""The per-element bound of the 1vsAll family (exact_oracle.OvaBound) and the constructions of
tests/test_gpu_one_vs_all_exact.py on the host: the bound holds for the oracles' own graphs evaluated in fp32, it
catches one (query, candidate) pair removed from the coldest row, the bit-exact tables meet their premise, and the
sweep's claimed geometry is the kernel's."""
import numpy as np
import pytest
import torch

import exact_oracle as xo
import k_vs_all_oracle
import one_vs_all_oracle
import relation_prediction_oracle
import test_gpu_one_vs_all_exact as gx


def _tables(model, E, R, k, rng, kind):
    K = xo.internal_k(model, k)
    if kind == "grid":
        return xo.grid_table(rng, E, K), xo.grid_table(rng, R, K)
    return rng.uniform(-0.5, 0.5, (E, K)).astype(np.float32), rng.uniform(-0.5, 0.5, (R, K)).astype(np.float32)


def _case(objective, model, kind, reduction, eps=0.0, E=300, R=40, k=16, B=200, seed=0):
    """(oracle float64, oracle float32, OvaBound with the fp32 graph's chains: one split, one query-tile range)."""
    rng = np.random.default_rng(seed)
    ent, rel = _tables(model, E, R, k, rng, kind)
    t = np.stack([rng.integers(0, E, B), rng.integers(0, R, B), rng.integers(0, E, B)], 1).astype(np.int32)
    labels = None
    bound = xo.OvaBound(model, ent, rel, t)
    if objective == "ova":
        run = lambda dt: one_vs_all_oracle.loss_and_grads(model, ent, rel, t, "s,o", reduction, matmul=True, dtype=dt)
        for side in ("s", "o"):
            bound.add_side(t, side, reduction, nsplit=1, xsplit=1)
    elif objective == "rel":
        run = lambda dt: relation_prediction_oracle.loss_and_grads(model, ent, rel, t, 0.5, reduction, matmul=True,
                                                                   dtype=dt)
        bound.add_side(t, "p", reduction, 0.5, nsplit=1, xsplit=1)
    else:
        labels = [sorted(set(rng.integers(0, E, rng.integers(1, 6)).tolist())) for _ in range(B)]
        t[:, 2] = [lab[0] for lab in labels]
        bound = xo.OvaBound(model, ent, rel, t)
        run = lambda dt: k_vs_all_oracle.loss_and_grads(model, ent, rel, t, labels, "o", reduction, eps, matmul=True,
                                                        dtype=dt)
        bound.add_side(t, "o", reduction, labels=labels, eps=eps, nsplit=1, xsplit=1)
    return run(torch.float64), run(torch.float32), bound, (ent, rel, t, labels)


CASES = [(obj, model, kind, red) for obj in ("ova", "kva", "rel") for model in ("DistMult", "ComplEx", "HolE")
         for kind in ("uniform", "grid") for red in ("sum", "mean")]


@pytest.mark.parametrize("objective,model,kind,reduction", CASES)
def test_bound_holds_for_the_fp32_graph(objective, model, kind, reduction):
    (l64, ge, gr), (l32, ge32, gr32), bound, _ = _case(objective, model, kind, reduction, 0.1 if objective == "kva" else 0.0)
    bound.check(ge32, gr32, ge, gr, (objective, model, kind, reduction))
    bound.check_loss(l32, l64, (objective, model, kind, reduction))


def _pair_term(objective, model, ent, rel, t, labels, reduction):
    """(row, term): the largest single (query, candidate) dX term of the coldest candidate row with a gradient, among the
    rows the batch does not look up (fed by the dX pass alone)."""
    E = torch.as_tensor(ent, dtype=torch.float64)
    R = torch.as_tensor(rel, dtype=torch.float64)
    tt = torch.as_tensor(t, dtype=torch.long)
    if objective == "rel":
        q = relation_prediction_oracle.relation_query(model, E[tt[:, 0]], E[tt[:, 2]])
        X, target = R, tt[:, 1]
    else:
        q = one_vs_all_oracle.query_vectors(model, "o", E[tt[:, 0]], R[tt[:, 1]], E[tt[:, 2]])
        X, target = E, tt[:, 2]
    lg = (q @ X.T).requires_grad_(True)
    if objective == "kva":
        loss = k_vs_all_oracle.side_loss(lg, k_vs_all_oracle.targets(labels, X.shape[0], 0.0), reduction).sum()
    else:
        loss = one_vs_all_oracle.side_loss(lg, target, reduction).sum() * (0.5 if objective == "rel" else 1.0)
    g = torch.autograd.grad(loss, lg)[0]
    terms = g[:, :, None] * q[:, None, :]  # [b, e, K]: the pair's contribution to row e
    size = terms.abs().amax(2)
    rows = terms.sum(0).abs().amax(1)
    touched = rows > 0
    touched[torch.unique(tt[:, 1] if objective == "rel" else tt[:, [0, 2]].reshape(-1))] = False
    e = int(torch.where(touched, rows, torch.full_like(rows, np.inf)).argmin())
    b = int(size[:, e].argmax())
    return e, terms[b, e].numpy()


@pytest.mark.parametrize("objective", ["ova", "kva", "rel"])
def test_bound_catches_one_pair_removed_from_the_coldest_row(objective):
    """The oracle's gradient with one (query, candidate) term taken out of the coldest candidate row violates the
    bound (U(-0.1, 0.1) tables as in the FB15k-237-shape tests: logits near 0, every non-target pair cold)."""
    model, reduction = "ComplEx", "sum"
    rng = np.random.default_rng(3)
    E, R, k, B = 2000, 300, 16, 300
    K = xo.internal_k(model, k)
    ent = rng.uniform(-0.1, 0.1, (E, K)).astype(np.float32)
    rel = rng.uniform(-0.1, 0.1, (R, K)).astype(np.float32)
    t = np.stack([rng.integers(0, E, B), rng.integers(0, R, B), rng.integers(0, E, B)], 1).astype(np.int32)
    labels = None
    bound = xo.OvaBound(model, ent, rel, t)
    if objective == "kva":
        labels = [sorted(set(rng.integers(0, E, rng.integers(1, 6)).tolist())) for _ in range(B)]
        t[:, 2] = [lab[0] for lab in labels]
        bound = xo.OvaBound(model, ent, rel, t)
        _, ge, gr = k_vs_all_oracle.loss_and_grads(model, ent, rel, t, labels, "o", reduction, matmul=True)
        bound.add_side(t, "o", reduction, labels=labels)
    elif objective == "rel":
        _, ge, gr = relation_prediction_oracle.loss_and_grads(model, ent, rel, t, 0.5, reduction, matmul=True)
        bound.add_side(t, "p", reduction, 0.5)
    else:
        _, ge, gr = one_vs_all_oracle.loss_and_grads(model, ent, rel, t, "o", reduction, matmul=True)
        bound.add_side(t, "o", reduction)
    bound.check(ge, gr, ge, gr)  # the oracle itself is within
    row, term = _pair_term(objective, model, ent, rel, t, labels, reduction)
    table = (gr if objective == "rel" else ge).copy()
    table[row] -= term
    with pytest.raises(AssertionError, match="worst error"):
        if objective == "rel":
            bound.check(ge, table, ge, gr)
        else:
            bound.check(table, gr, ge, gr)


def _within_2m40(want):
    """The oracle lies within 2^-40 of its largest entry of the fp32 values the GPU test compares with, and those are
    the oracle's own fp32 rounding wherever the oracle is not a residue below that unit."""
    want = np.asarray(want, np.float64)
    snapped = gx.exact_value(want).astype(np.float64)
    top = np.abs(want).max()
    return (np.abs(want - snapped).max() <= 2.0 ** -40 * top
            and np.array_equal(snapped[np.abs(want) > 2.0 ** -40 * top],
                               want.astype(np.float32).astype(np.float64)[np.abs(want) > 2.0 ** -40 * top]))


@pytest.mark.parametrize("case", gx.EXACT_OVA, ids=["-".join(map(str, c)) for c in gx.EXACT_OVA])
def test_bit_exact_one_vs_all_premise(case):
    model, k, G, g, B = case
    rng = np.random.default_rng(G * g + B)
    ent, rel, t = gx._exact_ova_case(model, k, G, g, B, 4, rng)
    live = (G - 1) * g
    assert live & (live - 1) == 0
    group = np.repeat(np.arange(G), g)
    assert (group[t[:, 0]] != group[t[:, 2]]).all()
    E = torch.as_tensor(ent, dtype=torch.float64)
    R = torch.as_tensor(rel, dtype=torch.float64)
    tt = torch.as_tensor(t, dtype=torch.long)
    for side in ("s", "o"):
        logits = one_vs_all_oracle.query_vectors(model, side, E[tt[:, 0]], R[tt[:, 1]], E[tt[:, 2]]) @ E.T
        assert bool(((logits == 0) | (logits == -128)).all())
        assert bool(((logits == 0).sum(1) == live).all())
    loss, ge, gr = one_vs_all_oracle.loss_and_grads(model, ent, rel, t, "s,o", "sum", matmul=True)
    assert _within_2m40(ge) and _within_2m40(gr)
    assert loss == pytest.approx(2 * B * np.log(live), rel=1e-12)


@pytest.mark.parametrize("case", gx.EXACT_KVA, ids=["-".join(map(str, c)) for c in gx.EXACT_KVA])
def test_bit_exact_k_vs_all_premise(case):
    model, k, G, g, B, reduction, eps = case
    rng = np.random.default_rng(G * g + B)
    E = G * g
    if reduction == "mean" or eps > 0:
        assert E & (E - 1) == 0
    ent, rel = gx.gated_tables(model, k, G, np.repeat(np.arange(G), g), 4, rng)
    labels = gx._labels(E, B, rng)
    q = gx._queries("o", labels, E, 4, rng)
    _, ge, gr = k_vs_all_oracle.loss_and_grads(model, ent, rel, q, labels, "o", reduction, eps, matmul=True)
    xo.assert_fp32_exact(torch.as_tensor(ge), "g_ent")
    xo.assert_fp32_exact(torch.as_tensor(gr), "g_rel")
    assert _within_2m40(ge) and _within_2m40(gr)


@pytest.mark.parametrize("model,k,B,n_live,G", gx.EXACT_REL)
def test_bit_exact_relation_premise(model, k, B, n_live, G):
    rng = np.random.default_rng(B + n_live)
    ent, rel, t = gx.exact_relation_case(model, k, B, rng, n_live, G)
    E = torch.as_tensor(ent, dtype=torch.float64)
    R = torch.as_tensor(rel, dtype=torch.float64)
    tt = torch.as_tensor(t, dtype=torch.long)
    logits = relation_prediction_oracle.relation_logits(model, E[tt[:, 0]], E[tt[:, 2]], R, matmul=True)
    assert bool(((logits == 0) | (logits == -128)).all())
    assert bool(((logits == 0).sum(1) == n_live).all())
    assert bool((logits.gather(1, tt[:, 1:2]) == 0).all())  # the positive's own relation is live
    loss, ge, gr = relation_prediction_oracle.loss_and_grads(model, ent, rel, t, 0.5, matmul=True)
    assert _within_2m40(ge) and _within_2m40(gr)


def test_sweep_geometry_is_the_kernels():
    for _, objective, model, k, E, R, B, geometry in gx.SWEEP:
        ns, xs = xo.ova_geometry(B, R if objective == "rel" else E, objective == "rel")
        ld = xo.row_stride(model, xo.internal_k(model, k))
        assert (ns, xs, -(-ld // 32)) == geometry, (objective, model, k, E, R, B)
    # what the sweep claims to cover
    claims = {c[0]: c[-1] for c in gx.SWEEP}
    assert claims["nsplit64-uneven"][0] == 64 and (2100 + 31) // 32 % 64 != 0
    assert claims["nsplit1-8500"][0] == 1 and -(-8500 // 32) > 264
    assert claims["rel-xsplit1"][1] == 1 and claims["rel-xsplit"][1] > 1 and claims["rel-nsplit64"][0] == 64
    assert {c[-1][2] for c in gx.SWEEP} >= {1, 2, 3, 4}


def test_clip_tables_give_the_edge_logits():
    ent, rel = gx.clip_tables()
    E = torch.as_tensor(ent, dtype=torch.float64)
    R = torch.as_tensor(rel, dtype=torch.float64)
    n = len(gx.CLIP_TARGETS)
    want = torch.tensor(gx.CLIP_TARGETS, dtype=torch.float64)
    for s_row in (0, 1):
        sign = 1.0 if s_row == 0 else -1.0
        q = one_vs_all_oracle.query_vectors("DistMult", "o", E[[s_row]], R[[0]], E[[2]])
        assert torch.equal((q @ E.T)[0, 3:3 + n], sign * want)
        qp = relation_prediction_oracle.relation_query("DistMult", E[[s_row]], E[[0]])
        assert torch.equal((qp @ R.T)[0, 1:1 + n], sign * want)
