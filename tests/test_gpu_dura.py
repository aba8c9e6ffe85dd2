"""The DURA regulariser on the GPU (kge_dura_step, DESIGN.md 3.16) against the float64 oracle of tests/dura_oracle.py.

- Exact tier: kge_dura_step alone on zeroed gradients, on tables with entries on the 2^-4 grid in [-1, 1] and
  power-of-two weights, so every square, product and partial sum is exact in fp32 in any RED order.  The gradient tables
  and the loss must equal the oracle's, pad columns and the rows outside the batch must stay 0.
- Bound tier: Glorot tables at the FB15k-237 shape, per element within dura_oracle.bound (its docstring derives it).
- Whole steps: sampled (non-deferred and deferred, bit-equal to each other and to the oracle after an exact SGD update),
  1vsAll with and without the relation term (exact_oracle.OvaBound plus the DURA bound), applied once per step.
- The looked-up-rows rule, the C-ABI's refusals, and fit end to end."""
import ctypes as C
import math
import zlib

import numpy as np
import pytest
import torch

import dura_oracle
import exact_oracle as xo
import one_vs_all_oracle
import relation_prediction_oracle
from ampligraph_b200 import _lib
from ampligraph_b200.engine import KGEEngine

pytestmark = pytest.mark.gpu

MODELS = ["DistMult", "ComplEx", "HolE"]


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a)).cuda().contiguous()


def dura_cfg(w_n, w_p):
    """The engine config of weights (w_n, w_p): lambda 1, alpha w_n, beta w_p (products exact)."""
    cfg = {"kind": "DURA", "lambda": 1.0, "alpha": w_n, "beta": w_p}
    return [cfg, dict(cfg)]


def grid16(rng, rows, K):
    """float32 [rows, K], entries on the 2^-4 grid in [-1, 1]."""
    return (rng.integers(-16, 17, (rows, K)) / 16.0).astype(np.float32)


def dense(eng, table):
    """padded [rows, ld] -> dense [rows, internal_k] float64 on the host, and whether every pad column is 0."""
    t = table.detach().cpu()
    k, kp = eng.k, eng.kp
    if eng.internal_k == k:
        return t[:, :k].double().numpy(), bool((t[:, k:] == 0).all())
    d = torch.cat([t[:, :k], t[:, kp:kp + k]], 1).double().numpy()
    return d, bool((t[:, k:kp] == 0).all()) and bool((t[:, kp + k:] == 0).all())


def _triples(E, R, B, rng):
    return np.stack([rng.integers(0, E, B), rng.integers(0, R, B), rng.integers(0, E, B)], 1).astype(np.int32)


def _run_alone(model, k, ent, rel, t, w_n, w_p):
    eng = KGEEngine(model, k, 1, ent.shape[0], rel.shape[0], regularizer=dura_cfg(w_n, w_p))
    eng.set_embeddings(ent, rel)
    eng.dura_backward(_dev(t), step=0)
    torch.cuda.synchronize()
    ge, pe = dense(eng, eng.g_ent)
    gr, pr = dense(eng, eng.g_rel)
    loss = eng.loss_acc.cpu().numpy().copy()
    launches = eng.launches
    eng.close()
    assert pe and pr, "pad columns of the gradient written"
    assert launches == (1 if len(t) else 0)
    return ge, gr, loss


# ---------------------------------------------------------------- exact tier
# k = 18: pad columns in the last float4 of each half; k = 36: kp = 36; "self-loop": h = t in every other positive;
# "repeated": one positive B times; "hot": entity 0 in every positive, as h, t or both
EXACT_CASES = [(m, k, E, R, B, shape, w) for m in MODELS
               for (k, E, R, B, shape) in [(16, 40, 5, 1, "B=1"), (16, 40, 5, 64, "repeated"), (8, 37, 3, 50, "self-loop"),
                                           (18, 33, 7, 300, "hot"), (36, 70, 4, 200, "kp=36")]
               for w in [(2.0 ** -3, 2.0 ** -5), (0.0, 2.0 ** -2), (2.0 ** -1, 0.0)]]


@pytest.mark.parametrize("model,k,E,R,B,shape,w", EXACT_CASES,
                         ids=["%s-%s-wn%g-wp%g" % (c[0], c[5], c[6][0], c[6][1]) for c in EXACT_CASES])
def test_exact_alone(model, k, E, R, B, shape, w):
    rng = np.random.default_rng(zlib.crc32(repr((model, shape, w)).encode()))
    K = xo.internal_k(model, k)
    ent, rel = grid16(rng, E, K), grid16(rng, R, K)
    t = _triples(E - 5, R, B, rng)  # the last five entity rows are never used
    if shape == "repeated":
        t[:] = t[0]
    if shape == "self-loop":
        t[::2, 2] = t[::2, 0]
    if shape == "hot":
        t[::3, 0] = 0
        t[1::3, 2] = 0
        t[2::3, [0, 2]] = 0
    ge, gr, loss = _run_alone(model, k, ent, rel, t, *w)
    want, we, wr = dura_oracle.loss_and_grads(model, ent, rel, t, *w)
    for name, x in (("g_ent", we), ("g_rel", wr)):
        xo.assert_fp32_exact(np.asarray(x), name)
    assert np.array_equal(ge, we) and np.array_equal(gr, wr), (np.abs(ge - we).max(), np.abs(gr - wr).max())
    assert loss[0] == 0.0 and loss[1] == want, (loss, want)
    assert not ge[E - 5:].any() and not ge[np.setdiff1d(np.arange(E), t[:, [0, 2]])].any()
    if w[1] == 0.0:
        assert not gr.any()
    else:
        assert not gr[np.setdiff1d(np.arange(R), t[:, 1])].any()


# ---------------------------------------------------------------- bound tier
@pytest.mark.parametrize("model", MODELS)
def test_bound_fb15k237(model):
    """Glorot tables at FB15k-237's shape, B = 27,212, k = 200."""
    E, R, B, k = 14541, 237, 27212, 200
    rng = np.random.default_rng(7)
    eng = KGEEngine(model, k, 1, E, R)
    eng.init_glorot_uniform(seed=3)
    ent, rel = (x.cpu().double().numpy() for x in eng.get_embeddings())
    eng.close()
    t = xo.zipf_triples(E, R, B, rng).astype(np.int32)
    w_n, w_p = 1e-3, 3e-3
    ge, gr, loss = _run_alone(model, k, ent.astype(np.float32), rel.astype(np.float32), t, w_n, w_p)
    want, we, wr = dura_oracle.loss_and_grads(model, ent, rel, t, w_n, w_p, device="cuda")
    lb, be, br = dura_oracle.bound(model, ent, rel, t, w_n, w_p)
    for name, got, w, b in (("g_ent", ge, we, be), ("g_rel", gr, wr, br)):
        err = np.abs(got - w)
        assert np.all(err <= b), (name, float((err / np.maximum(b, 1e-300)).max()))
    assert abs(loss[1] - want) <= lb, (loss[1], want, lb)
    assert np.count_nonzero(ge.any(1)) == len(np.unique(t[:, [0, 2]]))  # exactly the positives' rows


# ---------------------------------------------------------------- whole steps
@pytest.mark.parametrize("model,k", [("ComplEx", 16), ("DistMult", 33), ("HolE", 8)])
def test_sampled_step_deferred_and_not(model, k):
    """One sampled step with DURA, non-deferred and deferred: both equal x0 - lr (g_data + g_DURA) of the float64
    oracles bit for bit (SGD at lr = 2^-6 on exact gradients is exact), so they equal each other."""
    rng = np.random.default_rng(21)
    E, R, B, eta, lr, w = 500, 9, 1000, 4, 2.0 ** -6, (2.0 ** -6, 2.0 ** -7)
    K = xo.internal_k(model, k)
    ent, rel = xo.grid_table(rng, E, K), xo.grid_table(rng, R, K)
    t = xo.zipf_triples(E, R, B, rng)
    ne, nk = rng.integers(0, E, B * eta).astype(np.int32), rng.integers(0, 2, B * eta).astype(np.uint8)
    ref = xo.oracle_step(model, ent, rel, t, eta, ne, nk, loss="pairwise", loss_params={"margin": 1.0})
    dl, de, dr = dura_oracle.loss_and_grads(model, ent, rel, t, *w)
    want = [torch.as_tensor(x, dtype=torch.float64) - lr * (g.cpu() + torch.as_tensor(n))
            for x, g, n in ((ent, ref.g_ent, de), (rel, ref.g_rel, dr))]
    for x in want:
        xo.assert_fp32_exact(x, "updated table")
    got = {}
    for defer in (False, True):
        eng = KGEEngine(model, k, eta, E, R, loss="pairwise", loss_params={"margin": 1.0}, optimizer="sgd",
                        optimizer_params={"learning_rate": lr}, regularizer=dura_cfg(*w))
        eng.set_embeddings(ent, rel)
        assert int(eng.lib.kge_train_workspace_bytes(eng.h, B)) > 0
        eng.forward_backward(_dev(t), (_dev(ne), _dev(nk)), seed=0, step=0, defer=defer)
        assert eng._deferred == defer
        eng.dura_backward(_dev(t), step=0)  # accepted while the deferred step is pending
        eng.apply_gradients()
        acc = eng.loss_acc.cpu().numpy()
        assert acc[0] == ref.loss and acc[1] == dl, (acc, ref.loss, dl)
        got[defer] = (dense(eng, eng.ent)[0], dense(eng, eng.rel)[0])
        eng.close()
        for g, x in zip(got[defer], want):
            assert np.array_equal(g, x.numpy()), (defer, np.abs(g - x.numpy()).max())
    assert all(np.array_equal(a, b) for a, b in zip(got[False], got[True]))


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("rp_weight", [0.0, 0.5])
def test_one_vs_all_step(model, rp_weight):
    """A 1vsAll step (with the relation term or not) plus DURA against the 1vsAll oracle plus the DURA oracle; the DURA
    loss is counted once per step, not per side."""
    rng = np.random.default_rng(13)
    E, R, B, k, w = 300, 11, 200, 24, (0.01, 0.02)
    K = xo.internal_k(model, k)
    ent, rel = rng.uniform(-0.5, 0.5, (E, K)).astype(np.float32), rng.uniform(-0.5, 0.5, (R, K)).astype(np.float32)
    t = _triples(E, R, B, rng)
    t[1] = t[0]
    t[2, 2] = t[2, 0]
    eng = KGEEngine(model, k, 1, E, R, loss="multiclass_nll", regularizer=dura_cfg(*w))
    eng.set_embeddings(ent, rel)
    eng.one_vs_all_backward(_dev(t), "s,o", step=0)
    if rp_weight:
        eng.one_vs_all_relation_backward(_dev(t), rp_weight, step=0)
    eng.dura_backward(_dev(t), step=0)
    torch.cuda.synchronize()
    ge, gr = dense(eng, eng.g_ent)[0], dense(eng, eng.g_rel)[0]
    acc = eng.loss_acc.cpu().numpy()
    eng.close()
    if rp_weight:
        dl, de, dr = relation_prediction_oracle.loss_and_grads(model, ent, rel, t, rp_weight, "sum", sides="s,o")
    else:
        dl, de, dr = one_vs_all_oracle.loss_and_grads(model, ent, rel, t, "s,o", "sum")
    ob = xo.OvaBound(model, ent, rel, t)
    ob.add_side(t, "s")
    ob.add_side(t, "o")
    if rp_weight:
        ob.add_side(t, "p", weight=rp_weight)
    lb, be, br = dura_oracle.bound(model, ent, rel, t, *w)
    rl, re_, rr = dura_oracle.loss_and_grads(model, ent, rel, t, *w)
    # the DURA term's own bound, and one more rounding (u of the sum) where it is added to the data term's element
    for i, (b, n, d) in enumerate(((be, re_, de), (br, rr, dr))):
        ob.A[i] += torch.as_tensor(b / xo.FP32_EPS + np.abs(n) + np.abs(d), dtype=torch.float64)
    ob.check(ge, gr, de + re_, dr + rr, model)
    assert abs(acc[1] - rl) <= lb, (acc[1], rl, lb)
    ob.check_loss(acc[0], dl, model)


# ---------------------------------------------------------------- the looked-up-rows rule
@pytest.mark.parametrize("opt", ["adamax", "lazy_adam"])
def test_lazy_rule_untouched_rows_stay(opt):
    """With the looked-up-rows rule (optimizers.table_rules' outcome for Adamax with DURA, or lazy_), the rows the
    batch does not use keep their values and slots."""
    E, R, B, k = 200, 9, 30, 16
    rng = np.random.default_rng(2)
    t = _triples(E, R, B, rng)
    lazy = (True, True) if opt == "adamax" else None
    eng = KGEEngine("ComplEx", k, 1, E, R, optimizer=opt, regularizer=dura_cfg(0.1, 0.1), lazy_tables=lazy)
    eng.init_glorot_uniform(seed=1)
    e0, r0 = eng.ent.clone(), eng.rel.clone()
    s0 = [b.clone() for b in eng._sblocks if b is not None]
    eng.dura_backward(_dev(t), step=eng.t)
    eng.apply_gradients()
    for new, old, used, rows in ((eng.ent, e0, np.unique(t[:, [0, 2]]), E), (eng.rel, r0, np.unique(t[:, 1]), R)):
        moved = (new != old).any(1).cpu().numpy()
        assert moved[used].all()
        assert not moved[np.setdiff1d(np.arange(rows), used)].any()
    unused = np.concatenate([np.setdiff1d(np.arange(E), t[:, [0, 2]]), E + np.setdiff1d(np.arange(R), t[:, 1])])
    for s_new, s_old in zip([b for b in eng._sblocks if b is not None], s0):
        assert torch.equal(s_new[unused], s_old[unused])
    eng.close()


# ---------------------------------------------------------------- C ABI
def test_c_abi_refusals():
    lib = _lib.load()
    E, R, k = 50, 4, 8
    eng = KGEEngine("ComplEx", k, 1, E, R)
    eng.init_glorot_uniform(seed=1)
    t = _dev(np.array([[0, 1, 2], [3, 0, 4]], np.int32))
    P = lambda x: C.c_void_p(x.data_ptr()) if x is not None else C.c_void_p(0)
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    loss = torch.zeros(1, dtype=torch.float64, device="cuda")

    def call(e=eng, wn=0.1, wp=0.1, ent=eng.ent, rel=eng.rel, ge=eng.g_ent, gr=eng.g_rel, tr=t, B=2, lo=loss):
        return lib.kge_dura_step(e.h, wn, wp, P(ent), P(rel), P(ge), P(gr), P(tr), B, 0, P(lo), s)

    def last_error():
        return lib.kge_last_error().decode()
    INV, UNS = _lib.KGE_ERR_INVALID_ARGUMENT, _lib.KGE_ERR_UNSUPPORTED
    for model in ("TransE", "RotatE"):  # refused first, whatever else is wrong
        other = KGEEngine(model, k, 1, E, R)
        assert call(e=other, ent=other.ent, rel=other.rel, ge=other.g_ent, gr=other.g_rel) == UNS, model
        assert call(e=other, wn=-1.0, B=-1, tr=None) == UNS, model
        assert "TransE or RotatE" in last_error()
        other.close()
    for kw in (dict(wn=-1.0), dict(wp=-0.5), dict(wn=float("nan")), dict(wp=float("inf")), dict(wn=0.0, wp=0.0),
               dict(wn=-0.0, wp=0.0)):
        assert call(**kw, tr=None) == INV, kw  # the weights are checked before the pointers
        assert "weight_norm and weight_prod" in last_error(), kw
    assert call(B=-1, tr=None) == INV and "B < 0" in last_error()
    for kw in (dict(tr=None), dict(ent=None), dict(ge=None), dict(rel=None), dict(gr=None)):
        assert call(**kw) == INV, kw
        assert "null table, gradient or triples" in last_error(), kw
    torch.cuda.synchronize()
    assert float(loss) == 0.0 and not eng.g_ent.any() and not eng.g_rel.any()  # nothing was launched
    # w_p = 0: the relation table is not read and may be NULL; loss_dev may be NULL
    assert call(wp=0.0, rel=None, gr=None, lo=None) == 0
    # B = 0 is a no-op, with every pointer NULL
    assert call(B=0, tr=None, ent=None, rel=None, ge=None, gr=None, lo=None) == 0
    torch.cuda.synchronize()
    assert not eng.g_rel.any() and eng.g_ent.any()
    eng.close()


# ---------------------------------------------------------------- fit end to end
X_FIT = np.array([["e%d" % (i % 13), "r%d" % (i % 3), "e%d" % ((i * 7 + 3) % 13)] for i in range(40)])
LAM = 5e-2


def _reg():
    from ampligraph_b200.latent_features import regularizers
    return regularizers.DURA_regularizer({"lambda": LAM})


def _fit_model(reg, epochs, one_vs_all=None, loss="multiclass_nll", optimizer="adagrad", lr=0.1, batch_size=40):
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel, optimizers
    m = ScoringBasedEmbeddingModel(eta=2, k=8, scoring_type="ComplEx", seed=5)
    m.compile(optimizer=optimizers.get(optimizer, {"learning_rate": lr}), loss=loss, entity_relation_regularizer=reg)
    h = m.fit(X_FIT, batch_size=batch_size, epochs=epochs, verbose=False, one_vs_all=one_vs_all)
    return m, h


def _initial_tables(reg, loss="multiclass_nll"):
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    m = ScoringBasedEmbeddingModel(eta=2, k=8, scoring_type="ComplEx", seed=5)
    m.compile(optimizer="adagrad", loss=loss, entity_relation_regularizer=reg)
    t = m._index(X_FIT, fit=True)
    m.max_ent_size, m.max_rel_size = m.data_indexer.get_entities_count(), m.data_indexer.get_relations_count()
    m._build_engine()
    ent, rel = (x.cpu().double().numpy() for x in m.engine.get_embeddings())
    return ent, rel, t


def test_fit_one_vs_all_adagrad_against_oracle():
    """Two epochs of one full batch each, fit(one_vs_all='s,o') with Adagrad and DURA (lambda 5e-2): the tables follow
    the float64 oracle (1vsAll + DURA gradients, Keras's legacy Adagrad: a += g^2, x -= lr g / (sqrt(a) + 1e-7),
    a0 = 0.1), and the logged loss includes the DURA term."""
    lr = 0.1
    ent, rel, t = _initial_tables(_reg())
    m, h = _fit_model(_reg(), 2, one_vs_all="s,o", lr=lr)
    assert m.engine.dura_weights == (LAM, LAM)
    x = [ent.copy(), rel.copy()]
    a = [np.full_like(ent, 0.1), np.full_like(rel, 0.1)]
    losses = []
    for _ in range(2):
        dl, de, dr = one_vs_all_oracle.loss_and_grads("ComplEx", x[0], x[1], t, "s,o", "sum")
        rl, re_, rr = dura_oracle.loss_and_grads("ComplEx", x[0], x[1], t, LAM, LAM)
        losses.append(dl + rl)
        for i, g in enumerate((de + re_, dr + rr)):
            a[i] += g * g
            x[i] -= lr * g / (np.sqrt(a[i]) + 1e-7)
    got = [g.cpu().double().numpy() for g in m.engine.get_embeddings()]
    for g, w in zip(got, x):
        assert np.abs(g - w).max() <= 1e-5 * max(1.0, np.abs(w).max()), np.abs(g - w).max()
    assert h.history["loss"][-1] == pytest.approx(np.mean(losses), rel=1e-5)


def test_fit_sampled_loss_includes_dura():
    """A sampled fit with DURA runs; its logged loss after one step exceeds the same run's without DURA by the oracle's
    L_DURA of the initial tables (the data loss of step 0 is the same kernel on the same tables)."""
    ent, rel, t = _initial_tables(_reg(), loss="pairwise")
    _, h_on = _fit_model(_reg(), 1, loss="pairwise", optimizer="adam")
    _, h_off = _fit_model(None, 1, loss="pairwise", optimizer="adam")
    rl = dura_oracle.loss_and_grads("ComplEx", ent, rel, t, LAM, LAM)[0]
    lb = dura_oracle.bound("ComplEx", ent, rel, t, LAM, LAM)[0]
    diff = h_on.history["loss"][0] - h_off.history["loss"][0]
    assert rl > 0 and abs(diff - rl) <= lb + 4 * np.finfo(np.float64).eps * abs(h_on.history["loss"][0]), (diff, rl, lb)
    _, h2 = _fit_model(_reg(), 2, loss="pairwise", optimizer="adam", batch_size=16)
    assert all(math.isfinite(v) for v in h2.history["loss"])


def test_fit_one_vs_all_then_evaluate_predict_save(tmp_path):
    """The end-to-end use: compile with DURA, fit 1vsAll, then evaluate, predict and save_weights / load_weights as
    without a regulariser."""
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    m = ScoringBasedEmbeddingModel(eta=1, k=8, scoring_type="ComplEx", seed=5)
    m.compile(optimizer="adagrad", loss="multiclass_nll", entity_relation_regularizer=_reg())
    h = m.fit(X_FIT, batch_size=16, epochs=3, verbose=False, one_vs_all="s,o")
    assert all(math.isfinite(v) for v in h.history["loss"])
    ranks = np.asarray(m.evaluate(X_FIT[:10], use_filter={"train": X_FIT}, corrupt_side="s,o", verbose=False))
    assert ranks.shape == (10, 2) and (ranks >= 1).all() and (ranks <= 13).all()
    scores = np.asarray(m.predict(X_FIT[:10]))
    assert scores.shape == (10,) and np.isfinite(scores).all()
    path = str(tmp_path / "dura_model")
    m.save_weights(path)
    m2 = ScoringBasedEmbeddingModel(eta=1, k=8, scoring_type="ComplEx", seed=5)
    m2.compile(optimizer="adagrad", loss="multiclass_nll", entity_relation_regularizer=_reg())
    m2.load_weights(path)
    assert np.array_equal(np.asarray(m2.predict(X_FIT[:10])), scores)
