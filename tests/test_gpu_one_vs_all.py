"""1vsAll training on the GPU (kge_one_vs_all_step, DESIGN.md 3.12) against the float64 oracle of
tests/one_vs_all_oracle.py: loss and both gradient tables for DistMult, ComplEx and HolE on every side and reduction,
clipping, a million-entity overflow case, optimizer steps with the dense and the looked-up-rows rule, the FB15k-237
shape and the facade (the C-ABI's refusals: tests/test_gpu_all_candidates_abi.py).

Tolerance: per element, exact_oracle.OvaBound.  A gradient element is a sum over (query, entity) pairs of
g_be d l_be / d theta; the bound charges each pair the rounding of the fp32 chains it passes through (taken from the
kernel's split geometry), its logit's error ((ld + 4) 2^-24 sum_c |q_c x_c|) carried through the softmax, and the pair
in full where its logit is within that error of the clip.  A table-wide tolerance (1e-4 of the largest entry) would be
blind to cold rows: at n_ent = 14,541 one pair of a non-target row is about 7e-5 of a target row's entry, so a lost or
doubled pair, or a query lost from every non-target row, would pass.  The loss is held to the same analysis."""
import ctypes as C

import numpy as np
import pytest
import torch

import exact_oracle as xo
import one_vs_all_oracle
import optim_oracle
from ampligraph_b200 import _lib
from ampligraph_b200.engine import KGEEngine
from oracle import ref_step

pytestmark = pytest.mark.gpu

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
    return t


def _grads(eng):
    """The engine's gradient tables, unpacked to the dense [rows, internal_k] layout."""
    out = []
    for g, rows in ((eng.g_ent, eng.ent_rows), (eng.g_rel, eng.n_rel)):
        d = torch.empty((rows, eng.internal_k), dtype=torch.float32, device=eng.device)
        _lib.check(eng.lib.kge_unpack_rows(eng.h, C.c_void_p(g.data_ptr()), C.c_void_p(d.data_ptr()), rows, eng._stream()))
        out.append(d.cpu().numpy())
    return out


def _step(model, k, ent, rel, t, sides, reduction, optimizer="sgd", **kw):
    E, R = ent.shape[0], rel.shape[0]
    eng = KGEEngine(model, k, 1, E, R, loss="multiclass_nll", loss_params={"reduction": reduction}, optimizer=optimizer,
                    **kw)
    eng.set_embeddings(ent, rel)
    eng.one_vs_all_backward(_dev(t), sides)
    torch.cuda.synchronize()
    return eng


def _check(model, k, ent, rel, t, sides, reduction, device="cpu", matmul=False):
    eng = _step(model, k, ent, rel, t, sides, reduction)
    loss = float(eng.loss_acc[0])
    g_ent, g_rel = _grads(eng)
    want_loss, want_ent, want_rel = one_vs_all_oracle.loss_and_grads(model, ent, rel, t, sides, reduction, device, matmul)
    bound = xo.OvaBound(model, ent, rel, t, device)
    for side in sides.split(","):
        bound.add_side(t, side, reduction)
    bound.check_loss(loss, want_loss, (model, sides, reduction))
    bound.check(g_ent, g_rel, want_ent, want_rel, (model, sides, reduction))
    # pad columns of the gradient tables stay exactly 0
    assert bool((eng.g_ent[:, k:eng.kp] == 0).all()) and bool((eng.g_rel[:, k:eng.kp] == 0).all())
    eng.close()
    return want_ent


@pytest.mark.parametrize("shape", [(20, 37), (45, 70)])  # (n_ent, B): below one 32-entity tile / not a multiple of it
@pytest.mark.parametrize("reduction", ["sum", "mean"])
@pytest.mark.parametrize("sides", ["s,o", "o", "s"])
@pytest.mark.parametrize("model", ["DistMult", "ComplEx", "HolE"])
def test_matches_oracle(model, sides, reduction, shape):
    """k = 10 (pad columns), B not a multiple of the 32-query tile, repeated entities and relations within the batch."""
    rng = np.random.default_rng(11)
    E, B = shape
    R, k = 3, 10
    ent, rel = _tables(model, E, R, k, rng)
    _check(model, k, ent, rel, _triples(E, R, B, rng), sides, reduction)


@pytest.mark.parametrize("reduction", ["sum", "mean"])
def test_clipped_logits_have_zero_gradient(reduction):
    """Scaled DistMult tables: a good share of the logits leave [-75, 75] and contribute their clipped value to the
    loss and nothing to the gradient."""
    rng = np.random.default_rng(5)
    model, E, R, k, B = "DistMult", 40, 2, 8, 33
    ent, rel = _tables(model, E, R, k, rng, scale=1.0)
    ent *= 6.0
    rel *= 6.0
    t = _triples(E, R, B, rng)
    e_s, e_p, e_o = (torch.as_tensor(x, dtype=torch.float64) for x in (ent[t[:, 0]], rel[t[:, 1]], ent[t[:, 2]]))
    logits = ref_step.corruption_scores(model, "o", e_s, e_p, e_o, torch.as_tensor(ent, dtype=torch.float64))
    clipped = (logits.abs() > 75).double().mean()
    assert 0.05 < clipped < 0.8, clipped
    _check(model, k, ent, rel, t, "s,o", reduction)


def test_million_entities_near_the_clip_do_not_overflow():
    """n_ent = 10^6 logits near 75: sum_e exp(l_e) is about 10^6 e^75 > FLT_MAX, so only the max-subtracted sums give a
    finite loss; it equals the oracle's."""
    rng = np.random.default_rng(2)
    model, E, R, k, B = "DistMult", 1_000_000, 2, 4, 8
    ent = (1.0 + rng.uniform(-2e-3, 2e-3, (E, k))).astype(np.float32)
    rel = np.full((R, k), 18.74, np.float32)  # f = 4 * 18.74 * (1 +- 0.002)^2: within about 0.3 of 74.96
    t = _triples(E, R, B, rng)
    _check(model, k, ent, rel, t, "s,o", "sum", device="cuda", matmul=True)


@pytest.mark.parametrize("name,lazy", [("adam", (False, False)), ("adamax", (True, True))])
def test_optimizer_step(name, lazy):
    """One step of Adam (dense rule) and of Adamax with the looked-up-rows rule on both tables: every entity row and the
    batch's relation rows count as looked up; the other relation rows and their slots stay untouched."""
    rng = np.random.default_rng(8)
    model, E, R, k, B = "ComplEx", 50, 6, 10, 40
    ent, rel = _tables(model, E, R, k, rng)
    t = _triples(E, R, B, rng)
    t[:, 1] = np.where(t[:, 1] == 5, 4, t[:, 1])  # relation 5 is never looked up
    params = {"learning_rate": 0.01}
    eng = KGEEngine(model, k, 1, E, R, loss="multiclass_nll", optimizer=name, optimizer_params=params, lazy_tables=lazy)
    eng.set_embeddings(ent, rel)
    eng.one_vs_all_backward(_dev(t), "s,o", step=3)
    eng.apply_gradients()
    got_ent, got_rel = (x.cpu().numpy() for x in eng.get_embeddings())
    _, g_ent, g_rel = one_vs_all_oracle.loss_and_grads(model, ent, rel, t, "s,o", "sum")
    opt = optim_oracle.Optimizer(name, params["learning_rate"], lazy_tables={"ent": lazy[0], "rel": lazy[1]})
    want = {"ent": torch.as_tensor(ent).clone(), "rel": torch.as_tensor(rel).clone()}
    touched = {"ent": torch.arange(E), "rel": torch.as_tensor(t[:, 1], dtype=torch.long)}
    opt.step({key: (want[key], torch.as_tensor(g, dtype=torch.float32)) for key, g in (("ent", g_ent), ("rel", g_rel))},
             touched)
    for got, key in ((got_ent, "ent"), (got_rel, "rel")):
        assert np.allclose(got, want[key].numpy(), rtol=1e-5, atol=1e-6), (key, np.abs(got - want[key].numpy()).max())
    if lazy[0]:
        assert (eng.stamps["ent"] == _lib.load().kge_step_stamp(3)).all()
    eng.close()


def test_fb15k237_shape_against_device_oracle():
    """n_ent 14,541, 237 relations, ComplEx k = 200, B = 1,000, both sides, against the float64 oracle on the device."""
    rng = np.random.default_rng(1)
    model, E, R, k, B = "ComplEx", 14541, 237, 200, 1000
    ent, rel = _tables(model, E, R, k, rng, scale=0.1)
    _check(model, k, ent, rel, _triples(E, R, B, rng), "s,o", "sum", device="cuda", matmul=True)


def test_fit_one_vs_all():
    """fit(one_vs_all=...) on a small synthetic KG: the loss history (the running mean of the batch losses since the
    first step) decreases epoch by epoch, and the validation MRR is logged and about twice what random scores give
    (H_60 / 60 = 0.078); the model predicts and evaluates as usual afterwards."""
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel, optimizers
    rng = np.random.default_rng(0)
    E, R, n = 60, 3, 900
    s = rng.integers(0, E, n)
    r = rng.integers(0, R, n)
    o = (s * (r + 2) + 7) % E  # each (s, r) determines its object
    X = np.stack([s, r, o], 1).astype(str)
    X = np.unique(X, axis=0)
    valid = X[:30]
    for scoring, sides, reduction in (("ComplEx", "s,o", "sum"), ("DistMult", "o", "mean"), ("HolE", "s", "sum")):
        m = ScoringBasedEmbeddingModel(eta=5, k=32, scoring_type=scoring, seed=0)
        m.compile(optimizer=optimizers.OptimizerWrapper("adam", {"learning_rate": 0.03}), loss=_loss(reduction),
                  entity_relation_initializer="glorot_uniform")
        h = m.fit(X, batch_size=128, epochs=20, verbose=False, validation_data=valid, validation_freq=10,
                  validation_corrupt_side="o", one_vs_all=sides)
        losses = h.history["loss"]
        assert all(np.isfinite(losses)) and all(np.diff(losses) < 0) and losses[-1] < 0.9 * losses[0], (scoring, losses)
        assert "val_mrr" in h.history and h.history["val_mrr"][-1] > 0.15, (scoring, h.history["val_mrr"])
        ranks = m.evaluate(valid, corrupt_side="s,o")
        assert ranks.shape == (len(valid), 2)
        assert np.isfinite(m.predict(valid)).all()


def _loss(reduction):
    from ampligraph_b200.latent_features import loss_functions
    return loss_functions.get("multiclass_nll", {"reduction": reduction})
