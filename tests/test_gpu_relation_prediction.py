"""Relation prediction as an auxiliary 1vsAll objective on the GPU (kge_one_vs_all_relation_step, DESIGN.md 3.14)
against the float64 oracle of tests/relation_prediction_oracle.py: loss and both gradient tables for DistMult, ComplEx
and HolE under both reductions, relation counts below one tile, off the tile grid and at FB15k-237's 237 (split dX),
clipping, the term added to both entity sides, the weight's scaling, repeatability, the looked-up-rows optimizer rule,
the FB15k-237 shape and fit(relation_prediction_weight=...) (the C-ABI's refusals:
tests/test_gpu_all_candidates_abi.py).

Tolerance: per element, exact_oracle.OvaBound, as for the entity sides (tests/test_gpu_one_vs_all.py), with the
relation side's dX split over the query tiles (xsplit) in its chains and lambda in its weights."""
import ctypes as C

import numpy as np
import pytest
import torch

import exact_oracle as xo
import optim_oracle
import relation_prediction_oracle
from ampligraph_b200 import _lib
from ampligraph_b200.engine import KGEEngine, one_vs_all_splits

pytestmark = pytest.mark.gpu

RTOL = 1e-4


def _dev(a):
    return torch.as_tensor(a).cuda().contiguous()


def _tables(model, E, R, k, rng, scale=0.5):
    K = k if model == "DistMult" else 2 * k
    return rng.uniform(-scale, scale, (E, K)).astype(np.float32), rng.uniform(-scale, scale, (R, K)).astype(np.float32)


def _triples(E, R, B, rng):
    t = np.stack([rng.integers(0, E, B), rng.integers(0, R, B), rng.integers(0, E, B)], 1).astype(np.int32)
    t[1] = t[0]            # a repeated positive
    t[2, 0] = t[2, 2]      # a self-loop: the same entity on both sides
    t[3:6, 2] = t[3, 0]    # an entity repeated across positives and sides
    t[6:9, 1] = t[0, 1]    # a relation repeated across positives
    return t


def _grads(eng):
    """The engine's gradient tables, unpacked to the dense [rows, internal_k] layout."""
    out = []
    for g, rows in ((eng.g_ent, eng.ent_rows), (eng.g_rel, eng.n_rel)):
        d = torch.empty((rows, eng.internal_k), dtype=torch.float32, device=eng.device)
        _lib.check(eng.lib.kge_unpack_rows(eng.h, C.c_void_p(g.data_ptr()), C.c_void_p(d.data_ptr()), rows, eng._stream()))
        out.append(d.cpu().numpy())
    return out


def _close(got, want, rtol=RTOL):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    return np.abs(got - want).max() <= rtol * max(np.abs(want).max(), 1e-30)


def _engine(model, k, ent, rel, reduction="sum", **kw):
    eng = KGEEngine(model, k, 1, ent.shape[0], rel.shape[0], loss="multiclass_nll", loss_params={"reduction": reduction},
                    **kw)
    eng.set_embeddings(ent, rel)
    return eng


def _check(model, k, ent, rel, t, reduction, weight=1.0, sides=None, device="cpu", matmul=False):
    eng = _engine(model, k, ent, rel, reduction)
    td = _dev(t)
    if sides:
        eng.one_vs_all_backward(td, sides)
    eng.one_vs_all_relation_backward(td, weight)
    torch.cuda.synchronize()
    loss = float(eng.loss_acc[0])
    g_ent, g_rel = _grads(eng)
    want_loss, want_ent, want_rel = relation_prediction_oracle.loss_and_grads(model, ent, rel, t, weight, reduction,
                                                                              sides, device, matmul)
    bound = xo.OvaBound(model, ent, rel, t, device)
    for side in (sides.split(",") if sides else ()):
        bound.add_side(t, side, reduction)
    bound.add_side(t, "p", reduction, weight)
    bound.check_loss(loss, want_loss, (model, reduction, weight, sides))
    bound.check(g_ent, g_rel, want_ent, want_rel, (model, reduction, weight, sides))
    # pad columns of the gradient tables stay exactly 0
    assert bool((eng.g_ent[:, k:eng.kp] == 0).all()) and bool((eng.g_rel[:, k:eng.kp] == 0).all())
    eng.close()


@pytest.mark.parametrize("n_rel", [5, 45, 237])  # below one 32-relation tile / not a multiple of it / several splits
@pytest.mark.parametrize("reduction", ["sum", "mean"])
@pytest.mark.parametrize("model", ["DistMult", "ComplEx", "HolE"])
def test_matches_oracle(model, reduction, n_rel):
    """k = 10 (pad columns), B = 70 (not a multiple of the 32-query tile), repeated entities and relations."""
    rng = np.random.default_rng(11)
    E, B, k = 50, 70, 10
    ent, rel = _tables(model, E, n_rel, k, rng)
    if n_rel == 237:
        assert one_vs_all_splits(B, n_rel) > 1 and one_vs_all_splits(n_rel, B) > 1  # stats / dQ and dX both split
    _check(model, k, ent, rel, _triples(E, n_rel, B, rng), reduction, weight=0.5)


@pytest.mark.parametrize("reduction", ["sum", "mean"])
def test_clipped_logits_have_zero_gradient(reduction):
    """Scaled DistMult tables: a good share of the relation logits leave [-75, 75] and contribute their clipped value to
    the loss and nothing to the gradient."""
    rng = np.random.default_rng(5)
    model, E, R, k, B = "DistMult", 40, 40, 8, 33
    ent, rel = _tables(model, E, R, k, rng, scale=1.0)
    ent *= 6.0
    rel *= 6.0
    t = _triples(E, R, B, rng)
    e_s, e_o = (torch.as_tensor(x, dtype=torch.float64) for x in (ent[t[:, 0]], ent[t[:, 2]]))
    logits = relation_prediction_oracle.relation_logits(model, e_s, e_o, torch.as_tensor(rel, dtype=torch.float64))
    clipped = (logits.abs() > 75).double().mean()
    assert 0.05 < clipped < 0.8, clipped
    _check(model, k, ent, rel, t, reduction)


@pytest.mark.parametrize("model", ["DistMult", "ComplEx", "HolE"])
def test_added_to_both_entity_sides(model):
    """A 's,o' 1vsAll step followed by the relation step with lambda = 0.25 equals the oracle of
    L_s + L_o + lambda * L_p."""
    rng = np.random.default_rng(6)
    E, R, k, B = 70, 45, 10, 90
    ent, rel = _tables(model, E, R, k, rng)
    _check(model, k, ent, rel, _triples(E, R, B, rng), "sum", weight=0.25, sides="s,o")


def _relation_step(model, k, ent, rel, t, weight, reduction="sum"):
    eng = _engine(model, k, ent, rel, reduction)
    eng.one_vs_all_relation_backward(_dev(t), weight)
    torch.cuda.synchronize()
    out = float(eng.loss_acc[0]), eng.g_ent.clone(), eng.g_rel.clone()
    eng.close()
    return out


@pytest.mark.parametrize("reduction", ["sum", "mean"])
def test_weight_scales_exactly(reduction):
    """lambda = 2 gives twice lambda = 1's loss and gradients.  g_rel is summed in a fixed order, so scaling by a power
    of two is exact bit for bit; g_ent is added with red.global.add in no fixed order and compared to tolerance."""
    rng = np.random.default_rng(9)
    model, E, R, k, B = "ComplEx", 300, 237, 16, 200
    ent, rel = _tables(model, E, R, k, rng)
    t = _triples(E, R, B, rng)
    l1, ge1, gr1 = _relation_step(model, k, ent, rel, t, 1.0, reduction)
    l2, ge2, gr2 = _relation_step(model, k, ent, rel, t, 2.0, reduction)
    assert torch.equal(gr2, 2 * gr1)
    assert l2 == pytest.approx(2 * l1, rel=1e-12)
    assert _close(ge2.cpu().numpy(), 2 * ge1.cpu().numpy(), rtol=1e-6)


def test_relation_gradient_is_repeatable():
    rng = np.random.default_rng(10)
    model, E, R, k, B = "HolE", 500, 237, 24, 1000
    ent, rel = _tables(model, E, R, k, rng)
    t = _triples(E, R, B, rng)
    _, _, gr1 = _relation_step(model, k, ent, rel, t, 1.0)
    _, _, gr2 = _relation_step(model, k, ent, rel, t, 1.0)
    assert torch.equal(gr1, gr2)


def test_lazy_rule_stamps_every_relation_and_the_batch_entities():
    """Adamax with the looked-up-rows rule on both tables, the relation step alone: every relation row and exactly the
    batch's s and o rows are stamped and updated; the other entity rows and their slots stay untouched."""
    rng = np.random.default_rng(8)
    model, E, R, k, B = "ComplEx", 80, 40, 10, 40
    ent, rel = _tables(model, E, R, k, rng)
    t = _triples(E, R, B, rng)
    params = {"learning_rate": 0.01}
    eng = _engine(model, k, ent, rel, optimizer="adamax", optimizer_params=params, lazy_tables=(True, True))
    eng.one_vs_all_relation_backward(_dev(t), 1.0, step=3)
    eng.apply_gradients()
    got_ent, got_rel = (x.cpu().numpy() for x in eng.get_embeddings())
    _, g_ent, g_rel = relation_prediction_oracle.loss_and_grads(model, ent, rel, t, 1.0, "sum")
    opt = optim_oracle.Optimizer("adamax", params["learning_rate"], lazy_tables={"ent": True, "rel": True})
    want = {"ent": torch.as_tensor(ent).clone(), "rel": torch.as_tensor(rel).clone()}
    batch_ent = np.unique(t[:, [0, 2]])
    assert len(batch_ent) < E
    touched = {"ent": torch.as_tensor(batch_ent, dtype=torch.long), "rel": torch.arange(R)}
    opt.step({key: (want[key], torch.as_tensor(g, dtype=torch.float32)) for key, g in (("ent", g_ent), ("rel", g_rel))},
             touched)
    for got, key in ((got_ent, "ent"), (got_rel, "rel")):
        assert np.allclose(got, want[key].numpy(), rtol=1e-5, atol=1e-6), (key, np.abs(got - want[key].numpy()).max())
    stamp = _lib.load().kge_step_stamp(3)
    assert (eng.stamps["rel"] == stamp).all()
    stamped = (eng.stamps["ent"][:E] == stamp).cpu().numpy()
    assert np.array_equal(np.flatnonzero(stamped), batch_ent)
    untouched = np.setdiff1d(np.arange(E), batch_ent)
    assert np.array_equal(got_ent[untouched], ent[untouched])
    eng.close()


def test_fb15k237_shape_against_device_oracle():
    """n_ent 14,541, 237 relations, ComplEx k = 200, B = 1,000, against the float64 oracle on the device."""
    rng = np.random.default_rng(1)
    model, E, R, k, B = "ComplEx", 14541, 237, 200, 1000
    ent, rel = _tables(model, E, R, k, rng, scale=0.3)
    _check(model, k, ent, rel, _triples(E, R, B, rng), "sum", device="cuda", matmul=True)


def test_fit_relation_prediction():
    """fit(one_vs_all='s,o', relation_prediction_weight=1.0) on a small synthetic KG where (s, o) determines the
    relation: the loss history decreases epoch by epoch, and the filtered evaluate(corrupt_side='p') on the training
    triples gives an MRR well above what random scores give (H_8 / 8 = 0.34 over 8 relations).  The threshold is 0.8;
    on an H100 the fitted model ranks every probe triple's relation first (MRR 1.0).  predict and evaluate work
    afterwards."""
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel, loss_functions, optimizers
    rng = np.random.default_rng(0)
    E, R, n = 60, 8, 900
    s = rng.integers(0, E, n)
    o = rng.integers(0, E, n)
    r = (3 * s + 5 * o) % R  # each (s, o) determines its relation
    X = np.unique(np.stack([s, r, o], 1).astype(str), axis=0)
    probe = X[:200]
    m = ScoringBasedEmbeddingModel(eta=5, k=32, scoring_type="ComplEx", seed=0)
    m.compile(optimizer=optimizers.OptimizerWrapper("adam", {"learning_rate": 0.03}),
              loss=loss_functions.get("multiclass_nll", {"reduction": "sum"}), entity_relation_initializer="glorot_uniform")
    h = m.fit(X, batch_size=128, epochs=20, verbose=False, one_vs_all="s,o", relation_prediction_weight=1.0)
    losses = h.history["loss"]
    assert all(np.isfinite(losses)) and all(np.diff(losses) < 0) and losses[-1] < 0.9 * losses[0], losses
    ranks = m.evaluate(probe, use_filter={"train": X}, corrupt_side="p", verbose=False)
    assert ranks.shape == (len(probe), 1) and (ranks >= 1).all()
    mrr = float(np.mean(1.0 / ranks))
    print("filtered relation-prediction MRR on the training triples: %.3f" % mrr)
    assert mrr > 0.8, mrr
    assert np.isfinite(m.predict(probe)).all()
    assert m.evaluate(probe, corrupt_side="s,o", verbose=False).shape == (len(probe), 2)
