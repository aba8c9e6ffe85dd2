"""KvsAll training on the GPU (kge_k_vs_all_step, DESIGN.md 3.13) against the float64 oracle of
tests/k_vs_all_oracle.py: loss and both gradient tables for DistMult, ComplEx and HolE on both sides, both reductions,
with and without label smoothing; label sets on and across the 32-entity tile edges, up to every entity; clipping;
the looked-up-rows stamps and optimizer steps; the FB15k-237 shape; the facade (the C-ABI's refusals:
tests/test_gpu_all_candidates_abi.py).

Tolerance: per element, exact_oracle.OvaBound, as for 1vsAll (tests/test_gpu_one_vs_all.py): each (query, entity)
pair is charged the rounding of the fp32 chains it passes through, its logit's error carried through the sigmoid, a
few ulp of sigmoid - y, and in full where its logit is within that error of the clip.  A table-wide tolerance would be
blind to cold rows, where a single pair lies below 1e-4 of the largest entry.  The loss is held to the same
analysis."""
import ctypes as C

import numpy as np
import pytest
import torch

import exact_oracle as xo
import k_vs_all_oracle
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


def _labels(E, B, rng, special=True):
    """B label lists (sorted, distinct, in [0, E)): mostly 1-5 random labels; with `special`, also one label, 33
    labels, every entity, and pairs on the tile edges 31/32 and 63/64 where E reaches them."""
    labels = [sorted(set(rng.integers(0, E, rng.integers(1, 6)).tolist())) for _ in range(B)]
    if special:
        labels[0] = [int(rng.integers(0, E))]
        labels[1] = list(range(E))
        labels[2] = sorted(rng.choice(E, min(33, E), replace=False).tolist())
        labels[3] = [e for e in (0, 31, 32, 63, 64, E - 1) if e < E]
        labels[4] = [e for e in (30, 31) if e < E] or [E - 1]
        labels[5] = [e for e in (32, 33, 62, 63) if e < E] or [0]
    return labels


def _queries(side, labels, E, R, rng):
    """[B, 3] query rows: random kept entity and relation, the answer column holding the first label."""
    B = len(labels)
    keep, p = rng.integers(0, E, B), rng.integers(0, R, B)
    first = np.array([lab[0] for lab in labels])
    q = np.stack([keep, p, first], 1) if side == "o" else np.stack([first, p, keep], 1)
    q[1] = q[0]  # a repeated query row (with other labels): rows are independent
    return q.astype(np.int32)


def _csr(labels):
    off = np.concatenate([[0], np.cumsum([len(lab) for lab in labels])]).astype(np.int64)
    return off, np.concatenate(labels).astype(np.int32)


def _grads(eng):
    """The engine's gradient tables, unpacked to the dense [rows, internal_k] layout."""
    out = []
    for g, rows in ((eng.g_ent, eng.ent_rows), (eng.g_rel, eng.n_rel)):
        d = torch.empty((rows, eng.internal_k), dtype=torch.float32, device=eng.device)
        _lib.check(eng.lib.kge_unpack_rows(eng.h, C.c_void_p(g.data_ptr()), C.c_void_p(d.data_ptr()), rows, eng._stream()))
        out.append(d.cpu().numpy())
    return out


def _engine(model, k, ent, rel, reduction="sum", **kw):
    eng = KGEEngine(model, k, 1, ent.shape[0], rel.shape[0], loss="nll", loss_params={"reduction": reduction}, **kw)
    eng.set_embeddings(ent, rel)
    return eng


def _check(model, k, ent, rel, q, labels, side, reduction, eps, device="cpu", matmul=False, lo=0, hi=None):
    """One step over the query rows [lo, hi) of q (offsets sliced, ids shared: the offsets stay absolute)."""
    hi = len(q) if hi is None else hi
    off, ids = _csr(labels)
    eng = _engine(model, k, ent, rel, reduction, optimizer="sgd")
    eng.k_vs_all_backward(_dev(q[lo:hi]), side, _dev(off[lo:hi + 1]), _dev(ids), eps)
    torch.cuda.synchronize()
    loss = float(eng.loss_acc[0])
    g_ent, g_rel = _grads(eng)
    want_loss, want_ent, want_rel = k_vs_all_oracle.loss_and_grads(model, ent, rel, q[lo:hi], labels[lo:hi], side,
                                                                   reduction, eps, device, matmul)
    bound = xo.OvaBound(model, ent, rel, q[lo:hi], device)
    bound.add_side(q[lo:hi], side, reduction, labels=labels[lo:hi], eps=eps)
    bound.check_loss(loss, want_loss, (model, side, reduction, eps))
    bound.check(g_ent, g_rel, want_ent, want_rel, (model, side, reduction, eps))
    # pad columns of the gradient tables stay exactly 0
    assert bool((eng.g_ent[:, k:eng.kp] == 0).all()) and bool((eng.g_rel[:, k:eng.kp] == 0).all())
    eng.close()


@pytest.mark.parametrize("shape", [(20, 37), (45, 70)])  # (n_ent, B): below one 32-entity tile / not a multiple of it
@pytest.mark.parametrize("eps", [0.0, 0.1])
@pytest.mark.parametrize("reduction", ["sum", "mean"])
@pytest.mark.parametrize("side", ["o", "s"])
@pytest.mark.parametrize("model", ["DistMult", "ComplEx", "HolE"])
def test_matches_oracle(model, side, reduction, eps, shape):
    """k = 10 (pad columns), B not a multiple of the 32-query tile, queries with one label, 33 labels, every entity
    and labels on the tile edges."""
    rng = np.random.default_rng(11)
    E, B = shape
    R, k = 3, 10
    ent, rel = _tables(model, E, R, k, rng)
    labels = _labels(E, B, rng)
    _check(model, k, ent, rel, _queries(side, labels, E, R, rng), labels, side, reduction, eps)


@pytest.mark.parametrize("side", ["o", "s"])
def test_label_sets_across_tiles_and_splits(side):
    """n_ent = 5,000 (157 tiles, 64 entity splits of two or three tiles per query tile), 100 queries stepped as the
    slice [7, 90) of the label CSR: many labels per query, runs across tile and split edges, and every entity."""
    rng = np.random.default_rng(6)
    model, E, R, k = "ComplEx", 5000, 4, 12
    ent, rel = _tables(model, E, R, k, rng)
    labels = _labels(E, 100, rng)
    for i in range(10, 100, 9):
        labels[i] = sorted(set(rng.integers(0, E, int(rng.integers(30, 400))).tolist()))
    labels[8] = list(range(E))
    labels[9] = sorted(list(range(0, E, 32)) + list(range(31, E, 32)))
    labels[20] = list(range(100, 700))  # a run over about 19 tiles, across split boundaries
    _check(model, k, ent, rel, _queries(side, labels, E, R, rng), labels, side, "sum", 0.1, matmul=True, lo=7, hi=90)


@pytest.mark.parametrize("reduction", ["sum", "mean"])
def test_clipped_logits_have_zero_gradient(reduction):
    """Scaled DistMult tables: a good share of the logits leave [-75, 75] and contribute their clipped value to the
    loss and nothing to the gradient."""
    rng = np.random.default_rng(5)
    model, E, R, k, B = "DistMult", 40, 2, 8, 33
    ent, rel = _tables(model, E, R, k, rng, scale=1.0)
    ent *= 6.0
    rel *= 6.0
    labels = _labels(E, B, rng)
    q = _queries("o", labels, E, R, rng)
    e_s, e_p, e_o = (torch.as_tensor(x, dtype=torch.float64) for x in (ent[q[:, 0]], rel[q[:, 1]], ent[q[:, 2]]))
    logits = ref_step.corruption_scores(model, "o", e_s, e_p, e_o, torch.as_tensor(ent, dtype=torch.float64))
    clipped = (logits.abs() > 75).double().mean()
    assert 0.05 < clipped < 0.8, clipped
    _check(model, k, ent, rel, q, labels, "o", reduction, 0.1)


@pytest.mark.parametrize("name,lazy", [("adam", (False, False)), ("adamax", (True, True))])
def test_optimizer_step(name, lazy):
    """Both sides, then one step of Adam (dense rule) and of Adamax with the looked-up-rows rule on both tables: every
    entity row and the batch's relation rows are stamped; the other relation rows and their slots stay untouched."""
    rng = np.random.default_rng(8)
    model, E, R, k, B = "ComplEx", 50, 6, 10, 40
    ent, rel = _tables(model, E, R, k, rng)
    params = {"learning_rate": 0.01}
    eng = _engine(model, k, ent, rel, optimizer=name, optimizer_params=params, lazy_tables=lazy)
    g_ent, g_rel = np.zeros(ent.shape), np.zeros(rel.shape)
    used = []
    for side in ("o", "s"):
        labels = _labels(E, B, rng)
        q = _queries(side, labels, E, R, rng)
        q[:, 1] = np.where(q[:, 1] == 5, 4, q[:, 1])  # relation 5 is never looked up
        used.append(q[:, 1])
        off, ids = _csr(labels)
        eng.k_vs_all_backward(_dev(q), side, _dev(off), _dev(ids), 0.1, step=3)
        _, ge, gr = k_vs_all_oracle.loss_and_grads(model, ent, rel, q, labels, side, "sum", 0.1)
        g_ent, g_rel = g_ent + ge, g_rel + gr
    if lazy[0]:
        stamp = _lib.load().kge_step_stamp(3)
        assert (eng.stamps["ent"] == stamp).all()
        rel_stamped = (eng.stamps["rel"] == stamp).cpu().numpy()
        assert rel_stamped[np.concatenate(used)].all() and not rel_stamped[5]
    eng.apply_gradients()
    got_ent, got_rel = (x.cpu().numpy() for x in eng.get_embeddings())
    opt = optim_oracle.Optimizer(name, params["learning_rate"], lazy_tables={"ent": lazy[0], "rel": lazy[1]})
    want = {"ent": torch.as_tensor(ent).clone(), "rel": torch.as_tensor(rel).clone()}
    touched = {"ent": torch.arange(E), "rel": torch.as_tensor(np.concatenate(used), dtype=torch.long)}
    opt.step({key: (want[key], torch.as_tensor(g, dtype=torch.float32)) for key, g in (("ent", g_ent), ("rel", g_rel))},
             touched)
    for got, key in ((got_ent, "ent"), (got_rel, "rel")):
        assert np.allclose(got, want[key].numpy(), rtol=1e-5, atol=1e-6), (key, np.abs(got - want[key].numpy()).max())
    if lazy[1]:
        assert np.array_equal(got_rel[5], rel[5])
    eng.close()


def test_fb15k237_shape_against_device_oracle():
    """n_ent 14,541, 237 relations, ComplEx k = 200, 300 side-o queries with up to 60 labels each, against the float64
    oracle on the device."""
    rng = np.random.default_rng(1)
    model, E, R, k, B = "ComplEx", 14541, 237, 200, 300
    ent, rel = _tables(model, E, R, k, rng, scale=0.1)
    labels = [sorted(set(rng.integers(0, E, int(rng.integers(1, 61))).tolist())) for _ in range(B)]
    _check(model, k, ent, rel, _queries("o", labels, E, R, rng), labels, "o", "sum", 0.1, device="cuda", matmul=True)


def test_fit_k_vs_all_against_oracle():
    """fit(k_vs_all='s,o', label_smoothing=0.1) for two epochs with SGD on a small synthetic KG (repeated triples,
    several answers per query), with validation and EarlyStopping running inside it: the trained tables match the
    float64 oracle that runs the same grouping and step schedule (parallel.tables_close), and the validation metrics
    are logged."""
    from ampligraph_b200.latent_features import EarlyStopping, ScoringBasedEmbeddingModel, loss_functions, optimizers
    from ampligraph_b200.parallel import tables_close
    rng = np.random.default_rng(0)
    E, R, n, k, lr = 40, 3, 500, 8, 0.01
    t = np.stack([rng.integers(0, E, n), rng.integers(0, R, n), rng.integers(0, E, n)], 1)
    t[:E, 0] = np.arange(E)  # every entity and relation occurs
    t[:R, 1] = np.arange(R)
    t = np.concatenate([t, t[:50]])
    X = t.astype(str)
    valid = X[:20]
    for model, reduction in (("ComplEx", "sum"), ("DistMult", "mean")):
        m = ScoringBasedEmbeddingModel(eta=5, k=k, scoring_type=model, seed=0)
        K = m.internal_k
        ent0 = rng.uniform(-0.3, 0.3, (E, K)).astype(np.float32)
        rel0 = rng.uniform(-0.3, 0.3, (R, K)).astype(np.float32)
        m.compile(optimizer=optimizers.OptimizerWrapper("sgd", {"learning_rate": lr}),
                  loss=loss_functions.get("nll", {"reduction": reduction}), entity_relation_initializer=[ent0, rel0])
        es = EarlyStopping(monitor="val_mrr", patience=5)
        h = m.fit(X, batch_size=64, epochs=2, verbose=False, validation_data=valid, validation_freq=1,
                  callbacks=[es], k_vs_all="s,o", label_smoothing=0.1)
        assert len(h.history["val_mrr"]) == 2 and all(np.isfinite(h.history["loss"]))
        idx = m.get_indexes(X, "t", "raw2ind")  # the rows of ent0 / rel0 are these ids
        want_ent, want_rel = k_vs_all_oracle.fit_sgd(model, ent0, rel0, idx, "s,o", 64, 2, lr, reduction, 0.1)
        got_ent, got_rel = (x.cpu().numpy() for x in m.engine.get_embeddings())
        for got, want, init in ((got_ent, want_ent, ent0), (got_rel, want_rel, rel0)):
            ok, err = tables_close(got, want, init)
            assert ok, (model, err)
