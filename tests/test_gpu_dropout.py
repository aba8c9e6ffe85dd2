"""Embedding dropout of the all-candidate steps on the GPU (kge_set_embedding_dropout, fit(entity_dropout=...,
relation_dropout=...); DESIGN.md 3.19).

- Bound tier: 1vsAll, KvsAll and the relation side against the float64 oracle on the oracle's own dropped tables
  (tests/dropout_oracle.py), per element under exact_oracle.OvaBound plus the final scale rounding.
- Bit-exact tier: gated dyadic tables with p = 0.5 (scale 2): every operation is exact, so kernel and oracle agree
  element for element, which pins every mask bit the gradients read.
- Properties: p = (0, 0), p_rel = 0, the candidate mask's zero pattern, ranking untouched, refusals, the sizers.
- End to end: fit with dropout, then train_on_batch and evaluate."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import dropout_oracle as do
import exact_oracle as xo
from ampligraph_b200 import _lib
from ampligraph_b200.engine import (KGEEngine, k_vs_all_workspace_bytes, one_vs_all_relation_workspace_bytes,
                                    one_vs_all_workspace_bytes)

pytestmark = pytest.mark.gpu

SEED, STEP = 11, 5


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a)).cuda().contiguous()


def _grads(eng):
    out = []
    for g, rows in ((eng.g_ent, eng.ent_rows), (eng.g_rel, eng.n_rel)):
        d = torch.empty((rows, eng.internal_k), dtype=torch.float32, device=eng.device)
        _lib.check(eng.lib.kge_unpack_rows(eng.h, C.c_void_p(g.data_ptr()), C.c_void_p(d.data_ptr()), rows, eng._stream()))
        out.append(d.cpu().numpy())
    return out


def _csr(labels):
    off = np.concatenate([[0], np.cumsum([len(lab) for lab in labels])]).astype(np.int64)
    return off, np.concatenate(labels).astype(np.int32)


def _engine(objective, model, k, ent, rel, reduction="sum"):
    eng = KGEEngine(model, k, 1, ent.shape[0], rel.shape[0], loss="nll" if objective == "kva" else "multiclass_nll",
                    loss_params={"reduction": reduction}, optimizer="sgd")
    eng.set_embeddings(ent, rel)
    return eng


def _call(eng, objective, q, side, step=STEP, weight=0.5, labels=None, eps=0.0):
    if objective == "ova":
        eng.one_vs_all_backward(_dev(q), side, step=step)
    elif objective == "kva":
        off, ids = _csr(labels)
        eng.k_vs_all_backward(_dev(q), side, _dev(off), _dev(ids), eps, step=step)
    else:
        eng.one_vs_all_relation_backward(_dev(q), weight, step=step)


def _run(objective, model, k, ent, rel, q, side, reduction="sum", dropout=(0.4, 0.2), seed=SEED, step=STEP,
         weight=0.5, labels=None, eps=0.0):
    """One step on fresh gradient tables -> (loss, g_ent, g_rel); dropout None: never set."""
    eng = _engine(objective, model, k, ent, rel, reduction)
    if dropout is not None:
        eng.set_embedding_dropout(*dropout, seed=seed)
    _call(eng, objective, q, side, step, weight, labels, eps)
    torch.cuda.synchronize()
    loss = float(eng.loss_acc[0])
    g_ent, g_rel = _grads(eng)
    eng.close()
    return loss, g_ent, g_rel


def _sides(objective, side):
    return ["p"] if objective == "rel" else side.split(",")


def _oracle(objective, model, ent, rel, q, side, reduction, dr, weight=0.5, labels=None, eps=0.0):
    loss, g_ent, g_rel = 0.0, np.zeros(ent.shape), np.zeros(rel.shape)
    for sd in _sides(objective, side):
        lo, ge, gr, _ = do.side_step(model, ent, rel, q, sd, dr, reduction, weight if sd == "p" else 1.0, labels, eps)
        loss, g_ent, g_rel = loss + lo, g_ent + ge, g_rel + gr
    return loss, g_ent, g_rel


def _triples(E, R, B, rng):
    t = np.stack([rng.integers(0, E, B), rng.integers(0, R, B), rng.integers(0, E, B)], 1).astype(np.int32)
    if B > 3:
        t[1] = t[0]  # a repeated triple: its rows take two independent query masks
        t[2, 0] = t[2, 2]
    return t


def _labels(E, B, rng):
    labels = [sorted(set(rng.integers(0, E, rng.integers(1, 6)).tolist())) for _ in range(B)]
    if B > 1:
        labels[1] = [e for e in (0, 31, 32, 63, E - 1) if e < E]
    return labels


def _queries(side, labels, E, R, rng):
    B = len(labels)
    keep, p = rng.integers(0, E, B), rng.integers(0, R, B)
    first = np.array([lab[0] for lab in labels])
    q = np.stack([keep, p, first], 1) if side == "o" else np.stack([first, p, keep], 1)
    return q.astype(np.int32)


def _bound_check(objective, model, k, ent, rel, q, side, reduction="sum", dropout=(0.4, 0.2), labels=None, eps=0.0):
    got_loss, g_ent, g_rel = _run(objective, model, k, ent, rel, q, side, reduction, dropout, labels=labels, eps=eps)
    dr = do.Dropout(*dropout, SEED, STEP)
    want_loss, want_ent, want_rel = _oracle(objective, model, ent, rel, q, side, reduction, dr, labels=labels, eps=eps)
    bound = do.DropoutBound(model, ent, rel, q)
    for sd in _sides(objective, side):
        bound.add_dropout_side(q, sd, dr, reduction, 0.5 if sd == "p" else 1.0, labels, eps)
    where = (objective, model, k, side, reduction)
    bound.check_loss(got_loss, want_loss, where)
    bound.check(g_ent, g_rel, want_ent, want_rel, where)
    return g_ent, g_rel


# (id, objective, model, k, n_ent, n_rel, B, side): tile edges below and across 32 entities / queries
CASES = [
    ("ova-distmult-so", "ova", "DistMult", 36, 300, 5, 100, "s,o"),
    ("ova-complex-o", "ova", "ComplEx", 36, 300, 5, 100, "o"),
    ("ova-hole-s", "ova", "HolE", 16, 1007, 3, 70, "s"),
    ("ova-complex-below-tiles", "ova", "ComplEx", 10, 45, 3, 20, "s,o"),
    ("ova-distmult-n_ent31", "ova", "DistMult", 8, 31, 3, 33, "s,o"),
    ("kva-distmult-o", "kva", "DistMult", 12, 300, 5, 40, "o"),
    ("kva-complex-s", "kva", "ComplEx", 36, 300, 5, 100, "s"),
    ("kva-hole-o", "kva", "HolE", 16, 70, 3, 45, "o"),
    ("rel-distmult-xsplit1", "rel", "DistMult", 36, 50, 300, 32, None),
    ("rel-complex-xsplit", "rel", "ComplEx", 36, 50, 45, 200, None),
]


@pytest.mark.parametrize("reduction", ["sum", "mean"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_matches_oracle(case, reduction):
    _, objective, model, k, E, R, B, side = case
    rng = np.random.default_rng(k * 7919 + E + B)
    K = xo.internal_k(model, k)
    ent, rel = xo.grid_table(rng, E, K), xo.grid_table(rng, R, K)
    if objective == "kva":
        labels = _labels(E, B, rng)
        _bound_check("kva", model, k, ent, rel, _queries(side, labels, E, R, rng), side, reduction, labels=labels,
                     eps=0.1)
    else:
        _bound_check(objective, model, k, ent, rel, _triples(E, R, B, rng), side, reduction)


@pytest.mark.parametrize("objective,side", [("ova", "s,o"), ("kva", "o"), ("rel", None)])
def test_repeated_rows_take_their_own_masks(objective, side):
    """Every query of the batch is the same triple: the kernel meets the oracle, whose masks are keyed by the batch
    position, and those masks differ between the positions."""
    rng = np.random.default_rng(3)
    E, R, B, k = 80, 6, 40, 16
    ent, rel = xo.grid_table(rng, E, 2 * k), xo.grid_table(rng, R, 2 * k)
    q = np.tile(np.array([[3, 2, 7]], np.int32), (B, 1))
    labels = [[7]] * B if objective == "kva" else None
    _bound_check(objective, "ComplEx", k, ent, rel, q, side, labels=labels)
    f = do.Dropout(0.4, 0.2, SEED, STEP).factor("ComplEx", 2 * k, "o", 1, np.arange(B), "e")
    assert len({row.tobytes() for row in f}) == B


def test_label_smoothing_and_relation_weight_with_dropout():
    rng = np.random.default_rng(5)
    E, R, B, k = 200, 7, 64, 12
    ent, rel = xo.grid_table(rng, E, 2 * k), xo.grid_table(rng, R, 2 * k)
    labels = _labels(E, B, rng)
    _bound_check("kva", "ComplEx", k, ent, rel, _queries("s", labels, E, R, rng), "s", "mean", (0.3, 0.6), labels, 0.25)
    _bound_check("rel", "HolE", k, ent, rel, _triples(E, R, B, rng), None, "mean", (0.3, 0.6))


# --------------------------------------------------------------------------
# bit-exact tier
# --------------------------------------------------------------------------
def _gated(G, g, W, R, rng):
    """DistMult, k = G W: entity e is 1 on the W gate columns of its group e // g, every relation -128 on every gate
    column.  Under p = 0.5 a same-group logit is -1024 times the number of columns where s, p and x are all kept (so
    clipped unless there is none), every other logit exactly 0."""
    E = G * g
    ent = np.zeros((E, G * W), np.float32)
    for e in range(E):
        ent[e, (e // g) * W:(e // g + 1) * W] = 1.0
    rel = np.full((R, G * W), -128.0, np.float32)
    return ent, rel


def _snap(want):
    """The float64 oracle snapped to multiples of 2^-40 of its largest entry, as float32: on the gated tables every true
    value is such a multiple and fp32-exact, and the oracle's own residue (torch's logsumexp backward forms
    exp(l - log D), with log D rounded) is far below that unit."""
    want = np.asarray(want, np.float64)
    top = np.abs(want).max()
    if top == 0:
        return want.astype(np.float32)
    unit = 2.0 ** (np.ceil(np.log2(top)) - 40)
    snapped = np.round(want / unit) * unit
    return snapped.astype(np.float32)


def test_bit_exact_one_vs_all():
    """G = 5 groups of 16, W = 160: every row has 64 live candidates (the other groups) at logit 0, P = 1 / 64."""
    G, g, W, R, B = 5, 16, 160, 4, 100
    rng = np.random.default_rng(17)
    ent, rel = _gated(G, g, W, R, rng)
    E = G * g
    s = rng.integers(0, E, B)
    o = (s + g * rng.integers(1, G, B)) % E
    t = np.stack([s, rng.integers(0, R, B), o], 1).astype(np.int32)
    dr = do.Dropout(0.5, 0.5, SEED, STEP)
    for sd in ("s", "o"):  # the precondition: each row's same-group logits are clipped
        logits = do.side_step("DistMult", ent, rel, t, sd, dr)[3].numpy()
        assert ((logits == 0) | (logits <= -1024)).all() and ((logits == 0).sum(1) == 64).all()
    loss, g_ent, g_rel = _run("ova", "DistMult", G * W, ent, rel, t, "s,o", dropout=(0.5, 0.5))
    want_loss, want_ent, want_rel = _oracle("ova", "DistMult", ent, rel, t, "s,o", "sum", dr)
    assert np.array_equal(g_ent, _snap(want_ent)), np.abs(g_ent - want_ent).max()
    assert np.array_equal(g_rel, _snap(want_rel)), np.abs(g_rel - want_rel).max()
    assert want_loss == pytest.approx(2 * B * np.log(64), rel=1e-12) and loss == pytest.approx(want_loss, rel=1e-6)


@pytest.mark.parametrize("side", ["o", "s"])
@pytest.mark.parametrize("p", [0.5, 0.75])
def test_bit_exact_k_vs_all(side, p):
    """Live sigmoid 1/2 at logit 0: g = w (1/2 - y') is dyadic whatever the masks make live (eps = 1/2, n_ent 64)."""
    G, g, W, R, B = 4, 16, 8, 3, 70
    rng = np.random.default_rng(23)
    ent, rel = _gated(G, g, W, R, rng)
    E = G * g
    labels = _labels(E, B, rng)
    q = _queries(side, labels, E, R, rng)
    _, g_ent, g_rel = _run("kva", "DistMult", G * W, ent, rel, q, side, "mean", (p, p), labels=labels, eps=0.5)
    _, want_ent, want_rel = _oracle("kva", "DistMult", ent, rel, q, side, "mean", do.Dropout(p, p, SEED, STEP),
                                    labels=labels, eps=0.5)
    assert np.array_equal(g_ent, _snap(want_ent)), np.abs(g_ent - want_ent).max()
    assert np.array_equal(g_rel, _snap(want_rel)), np.abs(g_rel - want_rel).max()
    assert (g_ent != 0).any()  # the relation masks enter through q~ = s~ p~ and d/ds~ = p~ Gq


# --------------------------------------------------------------------------
# properties
# --------------------------------------------------------------------------
@pytest.mark.parametrize("objective,side", [("ova", "s,o"), ("kva", "s"), ("rel", None)])
def test_zero_dropout_is_the_plain_step(objective, side):
    """(0, 0) set, or set and cleared, gives loss and gradients bit-identical to a handle that never had dropout, with
    the same workspace size.  No row occurs twice in the batch, so no two red.global.add of the chain pass meet in
    one row and the plain step itself is reproducible bit for bit."""
    rng = np.random.default_rng(29)
    E, R, B, k = 300, 120, 100, 20
    ent, rel = xo.grid_table(rng, E, 2 * k), xo.grid_table(rng, R, 2 * k)
    perm = rng.permutation(E)
    q = np.stack([perm[:B], rng.permutation(R)[:B], perm[B:2 * B]], 1).astype(np.int32)
    labels = [[int(x)] for x in q[:, 0]] if objective == "kva" else None  # side s: the answer column 0
    plain = _run(objective, "ComplEx", k, ent, rel, q, side, dropout=None, labels=labels)
    zero = _run(objective, "ComplEx", k, ent, rel, q, side, dropout=(0.0, 0.0), labels=labels)
    eng = _engine(objective, "ComplEx", k, ent, rel)
    sizer = {"ova": eng.lib.kge_one_vs_all_workspace_bytes, "kva": eng.lib.kge_k_vs_all_workspace_bytes,
             "rel": eng.lib.kge_one_vs_all_relation_workspace_bytes}[objective]
    before = sizer(eng.h, B)
    eng.set_embedding_dropout(0.3, 0.2, seed=1)
    assert sizer(eng.h, B) > before
    eng.set_embedding_dropout(0.0, 0.0, seed=1)
    assert sizer(eng.h, B) == before
    _call(eng, objective, q, side, labels=labels)
    torch.cuda.synchronize()
    cleared = (float(eng.loss_acc[0]), *_grads(eng))
    eng.close()
    for other in (zero, cleared):
        assert other[0] == plain[0]
        assert np.array_equal(other[1], plain[1]) and np.array_equal(other[2], plain[2])


def test_relation_dropout_zero_leaves_relation_gradient_unmasked():
    """p_rel = 0: each relation row's gradient is that of the raw row (the oracle with scale 1 and no mask), and on the
    relation side every relation candidate row is fed."""
    rng = np.random.default_rng(31)
    E, R, B, k = 120, 30, 200, 16
    ent = xo.grid_table(rng, E, k, values=[-1.0, -0.5, 0.5, 1.0])
    rel = xo.grid_table(rng, R, k, values=[-1.0, -0.5, 0.5, 1.0])
    t = _triples(E, R, B, rng)
    g_ent, g_rel = _bound_check("rel", "DistMult", k, ent, rel, t, None, dropout=(0.5, 0.0))
    assert do.Dropout(0.5, 0.0, SEED, STEP).factor("DistMult", k, "p", 0, np.arange(R), "r").min() == 1.0
    zero_rows = (g_rel == 0).all(1)
    assert not zero_rows.any()


def test_candidate_mask_zero_pattern():
    """DistMult, side o, p_ent = 0.5: the gradient rows of candidates that are no query row are exactly zero where the
    side's candidate mask drops, a fraction within 5 sigma of p; the pattern differs between sides s and o and between
    two steps, and the same (seed, step) reproduces it bit for bit."""
    rng = np.random.default_rng(37)
    E, R, B, k, p = 2000, 4, 64, 64, 0.5
    ent = xo.grid_table(rng, E, k, values=[-1.0, -0.5, 0.5, 1.0])
    rel = xo.grid_table(rng, R, k, values=[-1.0, -0.5, 0.5, 1.0])
    t = np.stack([rng.integers(0, 10, B), rng.integers(0, R, B), rng.integers(0, 10, B)], 1).astype(np.int32)
    rows = slice(10, E)

    def zeros(side, step):
        return _run("ova", "DistMult", k, ent, rel, t, side, dropout=(p, 0.0), step=step)[1][rows] == 0

    z_o, z_s, z_o2, z_o_again = zeros("o", STEP), zeros("s", STEP), zeros("o", STEP + 1), zeros("o", STEP)
    n = z_o.size
    assert abs(z_o.mean() - p) <= 5 * math.sqrt(p * (1 - p) / n)
    want = ~do.Dropout(p, 0.0, SEED, STEP).factor("DistMult", k, "o", 0, np.arange(E), "e")[rows].astype(bool)
    assert np.array_equal(z_o, want)
    assert np.array_equal(z_o, z_o_again)
    assert not np.array_equal(z_o, z_s) and not np.array_equal(z_o, z_o2)


def test_ranking_and_scoring_ignore_dropout():
    rng = np.random.default_rng(41)
    E, R, B, k = 300, 6, 50, 16
    ent, rel = xo.grid_table(rng, E, 2 * k), xo.grid_table(rng, R, 2 * k)
    t = _dev(_triples(E, R, B, rng))
    eng = _engine("ova", "ComplEx", k, ent, rel)

    def outputs():
        out = [eng.score(t).cpu().numpy()]
        for side in ("s", "o", "p"):
            out.append(eng.rank(t, side).cpu().numpy())
        return out

    plain = outputs()
    eng.set_embedding_dropout(0.5, 0.5, seed=3)
    dropped = outputs()
    eng.close()
    for a, b in zip(plain, dropped):
        assert np.array_equal(a, b)


def test_sampled_step_refused_while_set():
    rng = np.random.default_rng(43)
    E, R, B, k = 100, 5, 32, 8
    ent, rel = xo.grid_table(rng, E, k), xo.grid_table(rng, R, k)
    eng = KGEEngine("DistMult", k, 2, E, R, loss="pairwise", optimizer="sgd")
    eng.set_embeddings(ent, rel)
    eng.set_embedding_dropout(0.2, 0.0, seed=0)
    t = _dev(_triples(E, R, B, rng))
    with pytest.raises(NotImplementedError, match="dropout"):
        eng.forward_backward(t, seed=0, step=0)
    eng.set_embedding_dropout(0.0, 0.0)
    eng.forward_backward(t, seed=0, step=0)
    torch.cuda.synchronize()
    eng.close()


def test_out_of_range_refused():
    eng = KGEEngine("DistMult", 8, 1, 10, 3, loss="multiclass_nll")
    for p_ent, p_rel in ((-0.1, 0.0), (0.0, 1.0), (1.5, 0.0), (float("nan"), 0.0), (0.0, float("-inf"))):
        assert eng.lib.kge_set_embedding_dropout(eng.h, p_ent, p_rel, 0) == _lib.KGE_ERR_INVALID_ARGUMENT
        with pytest.raises(ValueError, match="\\[0, 1\\)"):
            eng.set_embedding_dropout(p_ent, p_rel)
    assert eng.lib.kge_set_embedding_dropout(None, 0.1, 0.1, 0) == _lib.KGE_ERR_INVALID_ARGUMENT
    assert eng.lib.kge_set_embedding_dropout(eng.h, 0.0, 0.999, 0) == _lib.KGE_OK
    eng.close()


@pytest.mark.parametrize("model,k,E,R", [("DistMult", 36, 300, 5), ("ComplEx", 10, 14541, 237), ("HolE", 16, 45, 700)])
def test_sizers_match_the_engine_formulas(model, k, E, R):
    eng = KGEEngine(model, k, 1, E, R, loss="multiclass_nll")
    for on in (False, True, False):
        eng.set_embedding_dropout(0.25 if on else 0.0, 0.5 if on else 0.0, seed=9)
        for B in (1, 33, 1000):
            assert eng.lib.kge_one_vs_all_workspace_bytes(eng.h, B) == one_vs_all_workspace_bytes(B, E, eng.ld, on)
            assert eng.lib.kge_k_vs_all_workspace_bytes(eng.h, B) == k_vs_all_workspace_bytes(B, E, eng.ld, on)
            assert (eng.lib.kge_one_vs_all_relation_workspace_bytes(eng.h, B)
                    == one_vs_all_relation_workspace_bytes(B, R, eng.ld, on))
    eng.close()


# --------------------------------------------------------------------------
# end to end
# --------------------------------------------------------------------------
def _graph(rng, E=60, R=4, n=600):
    names = np.array(["e%d" % i for i in range(E)])
    return np.stack([names[rng.integers(0, E, n)], np.array(["r%d" % i for i in range(R)])[rng.integers(0, R, n)],
                     names[rng.integers(0, E, n)]], 1)


def _fit(X, training, dropout, reciprocal=True, epochs=12):
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    m = ScoringBasedEmbeddingModel(eta=1, k=16, scoring_type="ComplEx", seed=5, reciprocal_relations=reciprocal)
    m.compile(optimizer="adam", loss="multiclass_nll" if training == "one_vs_all" else "nll",
              entity_relation_regularizer="N3" if training == "one_vs_all" else None)
    kw = {"one_vs_all": "s,o"} if training == "one_vs_all" else {"k_vs_all": "s,o", "label_smoothing": 0.1}
    h = m.fit(X, batch_size=100, epochs=epochs, verbose=False, entity_dropout=dropout[0], relation_dropout=dropout[1],
              **kw)
    return m, h.history["loss"]


@pytest.mark.parametrize("training", ["one_vs_all", "k_vs_all"])
def test_fit_end_to_end(training):
    X = _graph(np.random.default_rng(47))
    m, loss = _fit(X, training, (0.4, 0.2))
    assert all(np.isfinite(loss)) and loss[-1] < loss[0]
    plain, _ = _fit(X, training, (0.0, 0.0))
    assert not np.array_equal(m.engine.ent.cpu().numpy(), plain.engine.ent.cpu().numpy())
    assert not np.array_equal(m.engine.rel.cpu().numpy(), plain.engine.rel.cpu().numpy())
    assert m.engine.dropout == (0.0, 0.0)
    ranks = m.evaluate(X[:20], corrupt_side="s,o", verbose=False)
    assert ranks.shape == (20, 2) and (ranks >= 1).all()
    # without reciprocal relations the model also trains on sampled batches after a fit with dropout
    m2, _ = _fit(X, training, (0.4, 0.2), reciprocal=False, epochs=2)
    if training == "one_vs_all":
        assert np.isfinite(m2.train_on_batch(X[:50]))
    assert m2.evaluate(X[:10], corrupt_side="s,o", verbose=False).shape == (10, 2)
