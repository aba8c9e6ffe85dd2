"""The N3 regulariser on the GPU (kge_n3_step, DESIGN.md 3.15) against the float64 oracle of tests/n3_oracle.py.

- Bit-exact tier: kge_n3_step alone on zeroed gradients, on tables whose every fp32 operation is exact (one-half
  entries in {0, +-1/2, +-1}; two-half pairs with exact moduli: one component 0, or (+-3/4, +-1), (+-3/8, +-1/2)) and
  lambda a power of two.  The gradient tables and the loss must equal the oracle's.
- Bound tier: Glorot tables at the FB15k-237 shape, per element within n3_oracle.bound (its docstring derives it).
- Whole steps: sampled (non-deferred and deferred, bit-equal to each other and to the oracle after an exact SGD
  update), 1vsAll with and without the relation term (exact_oracle.OvaBound plus the N3 bound), the two-phase step.
- The looked-up-rows rule, repeatability, the C-ABI's refusals, and fit end to end."""
import ctypes as C
import math
import zlib

import numpy as np
import pytest
import torch

import exact_oracle as xo
import n3_oracle
import one_vs_all_oracle
import relation_prediction_oracle
from ampligraph_b200 import _lib
from ampligraph_b200.engine import KGEEngine

pytestmark = pytest.mark.gpu

MODELS = ["TransE", "DistMult", "ComplEx", "HolE", "RotatE"]
PAIRS = [(0.0, 0.0), (0.0, 0.5), (0.0, -1.0), (1.0, 0.0), (-0.5, 0.0), (0.75, 1.0), (-0.75, 1.0), (1.0, -0.75),
         (0.375, 0.5), (-0.5, -0.375), (0.5, 0.375)]


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a)).cuda().contiguous()


def n3_cfg(lam_ent, lam_rel):
    return [{"kind": "N3", "lambda": lam_ent} if lam_ent else None, {"kind": "N3", "lambda": lam_rel} if lam_rel else None]


def exact_table(model, rng, rows, k):
    """float32 [rows, K] on which N3 is exact: {0, +-1/2, +-1} (one half), or pairs (x[d], x[k + d]) from PAIRS."""
    if model in n3_oracle.TWO_HALVES:
        idx = rng.integers(0, len(PAIRS), (rows, k))
        p = np.asarray(PAIRS)[idx]
        return np.concatenate([p[..., 0], p[..., 1]], 1).astype(np.float32)
    return rng.choice(np.array([-1.0, -0.5, 0.0, 0.5, 1.0]), (rows, k)).astype(np.float32)


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


def _run_alone(model, k, ent, rel, t, le, lr, zero=True):
    eng = KGEEngine(model, k, 1, ent.shape[0], rel.shape[0], regularizer=n3_cfg(le, lr))
    eng.set_embeddings(ent, rel)
    if not zero:
        eng.g_ent.copy_(torch.randn_like(eng.g_ent) * (eng.ent != 0))
        eng.g_rel.copy_(torch.randn_like(eng.g_rel) * (eng.rel != 0))
    eng.n3_backward(_dev(t), step=0)
    torch.cuda.synchronize()
    ge, pe = dense(eng, eng.g_ent)
    gr, pr = dense(eng, eng.g_rel)
    loss = eng.loss_acc.cpu().numpy().copy()
    eng.close()
    assert pe and pr, "pad columns of the gradient written"
    return ge, gr, loss


# ---------------------------------------------------------------- bit-exact tier
# "off the grids": 33 entity rows (not a multiple of the apply pass's 8 warps per CTA) and k = 18 (pad columns in the
# last float4 of each half); k = 36: kp = 36 = 4 (mod 32), so lane 0 takes a second chunk
EXACT_CASES = [(m, k, E, R, B, shape) for m in MODELS for (k, E, R, B, shape) in
               [(16, 40, 5, 1, "B=1"), (16, 40, 5, 64, "repeated"), (8, 37, 3, 50, "s=o"),
                (18, 33, 7, 300, "off the grids"), (36, 70, 4, 200, "kp=36")]]


@pytest.mark.parametrize("model,k,E,R,B,shape", EXACT_CASES, ids=["%s-%s" % (c[0], c[5]) for c in EXACT_CASES])
def test_exact_alone(model, k, E, R, B, shape):
    rng = np.random.default_rng(zlib.crc32(repr((model, shape)).encode()))
    ent, rel = exact_table(model, rng, E, k), exact_table(model, rng, R, k)
    t = _triples(E, R, B, rng)
    if shape == "repeated":
        t[:] = t[0]  # every row repeated
    if shape == "s=o":
        t[::2, 2] = t[::2, 0]  # an entity that is both s and o of one positive
    le, lr = 2.0 ** -3, (2.0 ** -5 if model != "RotatE" else 0.0)
    ge, gr, loss = _run_alone(model, k, ent, rel, t, le, lr)
    want, we, wr = n3_oracle.loss_and_grads(model, ent, rel, t, le, lr)
    for name, x in (("g_ent", we), ("g_rel", wr)):  # the loss is summed in fp64: exact, but not an fp32 value
        xo.assert_fp32_exact(np.asarray(x), name)
    assert np.array_equal(ge, we) and np.array_equal(gr, wr), (np.abs(ge - we).max(), np.abs(gr - wr).max())
    assert loss[0] == 0.0 and loss[1] == want, (loss, want)


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
    t = _triples(E, R, B, rng)
    le, lr = 1e-3, (3e-3 if model != "RotatE" else 0.0)
    ge, gr, loss = _run_alone(model, k, ent.astype(np.float32), rel.astype(np.float32), t, le, lr)
    want, we, wr = n3_oracle.loss_and_grads(model, ent, rel, t, le, lr, device="cuda")
    lb, be, br = n3_oracle.bound(model, ent, rel, t, le, lr, k)
    for name, got, w, b in (("g_ent", ge, we, be), ("g_rel", gr, wr, br)):
        err = np.abs(got - w)
        assert np.all(err <= b), (name, float((err / np.maximum(b, 1e-300)).max()))
    assert abs(loss[1] - want) <= lb, (loss[1], want, lb)
    assert np.count_nonzero(ge.any(1)) == len(np.unique(t[:, [0, 2]]))  # exactly the positives' rows


# ---------------------------------------------------------------- whole steps
def _sgd_engine(model, k, eta, E, R, lam, lr):
    return KGEEngine(model, k, eta, E, R, loss="pairwise", loss_params={"margin": 1.0}, optimizer="sgd",
                     optimizer_params={"learning_rate": lr}, regularizer=n3_cfg(lam, lam))


@pytest.mark.parametrize("model,k", [("ComplEx", 16), ("DistMult", 33), ("HolE", 8)])
def test_sampled_step_deferred_and_not(model, k):
    """One sampled step with N3, non-deferred and deferred: both equal x0 - lr (g_data + g_N3) of the float64 oracles
    bit for bit (SGD at lr = 2^-6 on exact gradients is exact), so they equal each other."""
    rng = np.random.default_rng(21)
    E, R, B, eta, lr, lam = 500, 9, 1000, 4, 2.0 ** -6, 2.0 ** -6
    ent, rel = exact_table(model, rng, E, k), exact_table(model, rng, R, k)
    t = xo.zipf_triples(E, R, B, rng)
    ne, nk = rng.integers(0, E, B * eta).astype(np.int32), rng.integers(0, 2, B * eta).astype(np.uint8)
    ref = xo.oracle_step(model, ent, rel, t, eta, ne, nk, loss="pairwise", loss_params={"margin": 1.0})
    n3l, n3e, n3r = n3_oracle.loss_and_grads(model, ent, rel, t, lam, lam)
    want = [torch.as_tensor(x, dtype=torch.float64) - lr * (g.cpu() + torch.as_tensor(n))
            for x, g, n in ((ent, ref.g_ent, n3e), (rel, ref.g_rel, n3r))]
    for w in want:
        xo.assert_fp32_exact(w, "updated table")
    got = {}
    for defer in (False, True):
        eng = _sgd_engine(model, k, eta, E, R, lam, lr)
        eng.set_embeddings(ent, rel)
        assert int(eng.lib.kge_train_workspace_bytes(eng.h, B)) > 0
        eng.forward_backward(_dev(t), (_dev(ne), _dev(nk)), seed=0, step=0, defer=defer)
        assert eng._deferred == defer
        eng.n3_backward(_dev(t), step=0)  # accepted while the deferred step is pending
        eng.apply_gradients()
        acc = eng.loss_acc.cpu().numpy()
        assert acc[0] == ref.loss and acc[1] == n3l, (acc, ref.loss, n3l)
        got[defer] = (dense(eng, eng.ent)[0], dense(eng, eng.rel)[0])
        eng.close()
        for g, w in zip(got[defer], want):
            assert np.array_equal(g, w.numpy()), (defer, np.abs(g - w.numpy()).max())
    assert all(np.array_equal(a, b) for a, b in zip(got[False], got[True]))


def test_two_phase_step():
    """The focusE / user-loss two-phase step adds N3 once: the tables equal x0 - lr (g_data + g_N3), g_data the
    oracle's under the dL/dscore the step passed to the kernel."""
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel, optimizers, regularizers
    from ampligraph_b200.latent_features.torch_losses import focuse_non_linearity
    rng = np.random.default_rng(4)
    model, k, E, R, B, eta, lr, lam = "DistMult", 16, 60, 5, 40, 2, 2.0 ** -6, 2.0 ** -4
    ent, rel = exact_table(model, rng, E, k), exact_table(model, rng, R, k)
    t = _triples(E, R, B, rng)
    m = ScoringBasedEmbeddingModel(eta=eta, k=k, scoring_type=model, seed=1)
    m.compile(optimizer=optimizers.get("sgd", {"learning_rate": lr}), loss="pairwise",
              entity_relation_regularizer=regularizers.N3_regularizer({"lambda": lam}))
    m.max_ent_size, m.max_rel_size = E, R
    m._build_engine()
    eng = m.engine
    eng.set_embeddings(ent, rel)
    m._focuse_nl, m._focuse_sw = focuse_non_linearity("linear"), 0.5
    seen = {}
    orig = eng.forward_backward

    def spy(triples, negatives=None, **kw):
        if kw.get("mode") == _lib.STEP_BACKWARD_EXT:
            seen.update(ne=negatives[0].cpu().numpy(), nk=negatives[1].cpu().numpy(), dpos=kw["dpos"].cpu().numpy(),
                        dneg=kw["dneg"].cpu().numpy())
        return orig(triples, negatives, **kw)
    eng.forward_backward = spy
    weights = _dev(rng.choice([0.0, 1.0], (B, 1)).astype(np.float32))
    m._two_phase_step(_dev(t), weights)
    ref = xo.oracle_step(model, ent, rel, t, eta, seen["ne"], seen["nk"], dpos=seen["dpos"], dneg=seen["dneg"])
    n3l, n3e, n3r = n3_oracle.loss_and_grads(model, ent, rel, t, lam, lam)
    for got, x, g, n in ((eng.ent, ent, ref.g_ent, n3e), (eng.rel, rel, ref.g_rel, n3r)):
        w = torch.as_tensor(x, dtype=torch.float64) - lr * (g.cpu() + torch.as_tensor(n))
        xo.assert_fp32_exact(w)
        assert np.array_equal(dense(eng, got)[0], w.numpy())
    assert float(eng.loss_acc[1]) == n3l


def _ova_bound_with_n3(model, ent, rel, t, lam, rp_weight, want_data):
    ob = xo.OvaBound(model, ent, rel, t)
    ob.add_side(t, "s")
    ob.add_side(t, "o")
    if rp_weight:
        ob.add_side(t, "p", weight=rp_weight)
    _, be, br = n3_oracle.bound(model, ent, rel, t, lam, lam, ent.shape[1] // 2)
    _, ne_, nr_ = n3_oracle.loss_and_grads(model, ent, rel, t, lam, lam)
    # the N3 term's own bound, and one more rounding (u of the sum) where it is added to the data term's element
    for i, (b, n, d) in enumerate(((be, ne_, want_data[0]), (br, nr_, want_data[1]))):
        ob.A[i] += torch.as_tensor(b / xo.FP32_EPS + np.abs(n) + np.abs(d), dtype=torch.float64)
    return ob, ne_, nr_


@pytest.mark.parametrize("model", ["DistMult", "ComplEx", "HolE"])
@pytest.mark.parametrize("rp_weight", [0.0, 0.5])
def test_one_vs_all_step(model, rp_weight):
    rng = np.random.default_rng(13)
    E, R, B, k, lam = 300, 11, 200, 24, 0.01
    K = xo.internal_k(model, k)
    ent, rel = rng.uniform(-0.5, 0.5, (E, K)).astype(np.float32), rng.uniform(-0.5, 0.5, (R, K)).astype(np.float32)
    t = _triples(E, R, B, rng)
    t[1] = t[0]
    eng = KGEEngine(model, k, 1, E, R, loss="multiclass_nll", regularizer=n3_cfg(lam, lam))
    eng.set_embeddings(ent, rel)
    eng.one_vs_all_backward(_dev(t), "s,o", step=0)
    if rp_weight:
        eng.one_vs_all_relation_backward(_dev(t), rp_weight, step=0)
    eng.n3_backward(_dev(t), step=0)
    torch.cuda.synchronize()
    ge, gr = dense(eng, eng.g_ent)[0], dense(eng, eng.g_rel)[0]
    acc = eng.loss_acc.cpu().numpy()
    eng.close()
    if rp_weight:
        dl, de, dr = relation_prediction_oracle.loss_and_grads(model, ent, rel, t, rp_weight, "sum", sides="s,o")
    else:
        dl, de, dr = one_vs_all_oracle.loss_and_grads(model, ent, rel, t, "s,o", "sum")
    ob, ne_, nr_ = _ova_bound_with_n3(model, ent, rel, t, lam, rp_weight, (de, dr))
    ob.check(ge, gr, de + ne_, dr + nr_, model)
    n3l = n3_oracle.loss_and_grads(model, ent, rel, t, lam, lam)[0]
    lb = n3_oracle.bound(model, ent, rel, t, lam, lam, k)[0]
    assert abs(acc[1] - n3l) <= lb, (acc[1], n3l, lb)  # counted once per step, not per side
    ob.check_loss(acc[0], dl, model)


# ---------------------------------------------------------------- the looked-up-rows rule, repeatability
@pytest.mark.parametrize("opt", ["adamax", "lazy_adam"])
def test_lazy_rule_untouched_rows_stay(opt):
    E, R, B, k = 200, 9, 30, 16
    rng = np.random.default_rng(2)
    t = _triples(E, R, B, rng)
    lazy = (True, True) if opt == "adamax" else None  # optimizers.table_rules' outcome for Adamax with N3 tables
    eng = KGEEngine("ComplEx", k, 1, E, R, optimizer=opt, regularizer=n3_cfg(0.1, 0.1), lazy_tables=lazy)
    eng.init_glorot_uniform(seed=1)
    e0, r0 = eng.ent.clone(), eng.rel.clone()
    eng.n3_backward(_dev(t), step=eng.t)
    eng.apply_gradients()
    for new, old, used, rows in ((eng.ent, e0, np.unique(t[:, [0, 2]]), E), (eng.rel, r0, np.unique(t[:, 1]), R)):
        moved = (new != old).any(1).cpu().numpy()
        assert moved[used].all()
        assert not moved[np.setdiff1d(np.arange(rows), used)].any()
    eng.close()


def test_repeatable():
    rng = np.random.default_rng(8)
    E, R, B, k = 3000, 40, 20000, 100
    eng = KGEEngine("ComplEx", k, 1, E, R, regularizer=n3_cfg(1e-3, 2e-3))
    eng.init_glorot_uniform(seed=2)
    t = _dev(_triples(E, R, B, rng))
    g0 = torch.randn_like(eng._gblock) * (eng._pblock != 0)
    out = []
    for _ in range(2):
        eng._gblock.copy_(g0)
        eng.n3_backward(t, step=0)
        out.append(eng._gblock.clone())
    assert torch.equal(out[0], out[1])
    eng.close()


# ---------------------------------------------------------------- C ABI
def test_c_abi_refusals():
    lib = _lib.load()
    E, R, k = 50, 4, 8
    eng = KGEEngine("ComplEx", k, 1, E, R)
    rot = KGEEngine("RotatE", k, 1, E, R)
    t = _dev(np.array([[0, 1, 2], [3, 0, 4]], np.int32))
    ws = torch.zeros(int(lib.kge_n3_workspace_bytes(eng.h)) + 16, dtype=torch.uint8, device="cuda")
    assert lib.kge_n3_workspace_bytes(eng.h) == eng.n3_workspace_bytes == (4 * (E + R) + 15) // 16 * 16
    P = lambda x: C.c_void_p(x.data_ptr()) if x is not None else C.c_void_p(0)
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    need = eng.n3_workspace_bytes

    def call(e=eng, le=0.1, lr=0.1, ent=eng.ent, rel=eng.rel, ge=eng.g_ent, gr=eng.g_rel, tr=t, B=2, w=P(ws), wb=need):
        return lib.kge_n3_step(e.h, le, lr, P(ent), P(rel), P(ge), P(gr), P(tr), B, 0, None, w, wb, s)
    INV, UNS = _lib.KGE_ERR_INVALID_ARGUMENT, _lib.KGE_ERR_UNSUPPORTED
    for kw in (dict(le=-1.0), dict(lr=float("nan")), dict(le=float("inf")), dict(le=0.0, lr=0.0), dict(B=-1),
               dict(tr=None), dict(ent=None), dict(gr=None), dict(w=C.c_void_p(0)), dict(wb=need - 1),
               dict(w=C.c_void_p(ws.data_ptr() + 4))):
        assert call(**kw) == INV, kw
    assert lib.kge_n3_step(rot.h, 0.0, 0.1, P(rot.ent), P(rot.rel), P(rot.g_ent), P(rot.g_rel), P(t), 2, 0, None,
                           P(ws), need, s) == UNS
    assert lib.kge_n3_step(rot.h, 0.1, 0.0, P(rot.ent), None, P(rot.g_ent), None, P(t), 2, 0, None, P(ws), need, s) == 0
    assert call(le=0.0, ent=None, ge=None) == 0  # a table whose lambda is 0 may be NULL
    assert call(B=0, tr=None, w=C.c_void_p(0), wb=0) == 0  # B = 0 is a no-op
    torch.cuda.synchronize()
    eng.close()
    rot.close()


# ---------------------------------------------------------------- fit end to end
X_FIT = np.array([["e%d" % (i % 13), "r%d" % (i % 3), "e%d" % ((i * 7 + 3) % 13)] for i in range(40)])


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
    """Two epochs of one full batch each, fit(one_vs_all='s,o') with Adagrad and ['N3', 'N3']: the tables follow the
    float64 oracle (1vsAll + N3 gradients, Keras's legacy Adagrad: a += g^2, x -= lr g / (sqrt(a) + 1e-7), a0 = 0.1),
    and the logged loss includes lambda L_N3 (lambda the default, 1e-3)."""
    lr = 0.1
    ent, rel, t = _initial_tables(["N3", "N3"])
    m, h = _fit_model(["N3", "N3"], 2, one_vs_all="s,o", lr=lr)
    assert m._regularizer[0].lam == m._regularizer[1].lam == 1e-3
    x = [ent.copy(), rel.copy()]
    a = [np.full_like(ent, 0.1), np.full_like(rel, 0.1)]
    losses = []
    for _ in range(2):
        dl, de, dr = one_vs_all_oracle.loss_and_grads("ComplEx", x[0], x[1], t, "s,o", "sum")
        nl, ne_, nr_ = n3_oracle.loss_and_grads("ComplEx", x[0], x[1], t, 1e-3, 1e-3)
        losses.append(dl + nl)
        for i, g in enumerate((de + ne_, dr + nr_)):
            a[i] += g * g
            x[i] -= lr * g / (np.sqrt(a[i]) + 1e-7)
    got = [g.cpu().double().numpy() for g in m.engine.get_embeddings()]
    for g, w in zip(got, x):
        assert np.abs(g - w).max() <= 1e-5 * max(1.0, np.abs(w).max()), np.abs(g - w).max()
    assert h.history["loss"][-1] == pytest.approx(np.mean(losses), rel=1e-5)


def test_fit_sampled_loss_includes_n3():
    """A sampled fit with N3 runs; its logged loss after one step exceeds the same run's without N3 by the oracle's
    L_N3 of the initial tables (the data loss of step 0 is the same kernel on the same tables)."""
    ent, rel, t = _initial_tables("N3", loss="pairwise")
    _, h_on = _fit_model("N3", 1, loss="pairwise", optimizer="adam")
    _, h_off = _fit_model(None, 1, loss="pairwise", optimizer="adam")
    n3l = n3_oracle.loss_and_grads("ComplEx", ent, rel, t, 1e-3, 1e-3)[0]
    lb = n3_oracle.bound("ComplEx", ent, rel, t, 1e-3, 1e-3, 8)[0]
    diff = h_on.history["loss"][0] - h_off.history["loss"][0]
    assert abs(diff - n3l) <= lb + 4 * np.finfo(np.float64).eps * abs(h_on.history["loss"][0]), (diff, n3l, lb)
    _, h2 = _fit_model("N3", 2, loss="pairwise", optimizer="adam", batch_size=16)
    assert all(math.isfinite(v) for v in h2.history["loss"])
