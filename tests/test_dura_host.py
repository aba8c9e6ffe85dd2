"""CPU tests of the DURA regulariser: the registry, the refusals (at compile, and before anything is indexed or trained),
the optimizer's per-table rule with DURA, the engine config, select_best_model_ranking's grid, the C-ABI entry point,
and the float64 oracle (tests/dura_oracle.py) against a numpy restatement, central differences and the closed form."""
import os
import re

import numpy as np
import pytest

import dura_oracle

X = np.array([["a", "r", "b"], ["b", "r", "c"], ["c", "q", "a"]])


def _model(scoring="ComplEx", loss="multiclass_nll", reg="DURA", optimizer="adam"):
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    m = ScoringBasedEmbeddingModel(eta=2, k=4, scoring_type=scoring)
    m.compile(optimizer=optimizer, loss=loss, entity_relation_regularizer=reg)
    return m


# ---------------------------------------------------------------- registry
def test_registry_names_and_defaults():
    from ampligraph_b200.latent_features import regularizers
    for name in ("DURA", "dura"):
        r = regularizers.get(name)
        assert isinstance(r, regularizers.DURARegularizer) and r.__name__ == "DURA"
        assert (r.lam, r.alpha, r.beta) == (1e-3, 1.0, 1.0)
        assert r.kernel_params() == {"kind": "DURA", "lambda": 1e-3, "alpha": 1.0, "beta": 1.0}
        assert regularizers.is_per_occurrence(r.kernel_params()) and not regularizers.is_n3(r.kernel_params())
    r = regularizers.get("DURA", {"lambda": 0.05, "beta": 0.0})
    assert (r.lam, r.alpha, r.beta) == (0.05, 1.0, 0.0)
    inst = regularizers.DURA_regularizer({"lambda": 0.25, "alpha": 0.5})
    assert regularizers.get(inst) is inst
    assert regularizers.get_pair(inst) == [inst, inst]
    assert regularizers.is_per_occurrence(regularizers.get("N3").kernel_params())
    assert not regularizers.is_per_occurrence(regularizers.get("LP").kernel_params())
    assert not regularizers.is_per_occurrence(None)


def test_registry_unchanged_for_other_names():
    from ampligraph_b200.latent_features import regularizers
    assert regularizers.get("l3").p == 3 and regularizers.get("N3").lam == 1e-3
    for bad in ("DURA2", "duality", {"class_name": "DURA"}):
        with pytest.raises(ValueError, match=re.escape("Could not interpret regularizer identifier: %r" % (bad,))):
            regularizers.get(bad)


@pytest.mark.parametrize("key", ["lambda", "alpha", "beta"])
@pytest.mark.parametrize("bad", [-1.0, float("nan"), float("inf"), float("-inf")])
def test_bad_parameter_refused(key, bad):
    from ampligraph_b200.latent_features import regularizers
    with pytest.raises(ValueError, match="DURA regularizer: %s must be finite and >= 0" % key):
        regularizers.DURA_regularizer({key: bad})


@pytest.mark.parametrize("params", [{"lambda": 0.0}, {"alpha": 0.0, "beta": 0.0}, {"lambda": 0.0, "alpha": 0.0}])
def test_both_weights_zero_refused(params):
    from ampligraph_b200.latent_features import regularizers
    with pytest.raises(ValueError, match="DURA regularizer: lambda \\* alpha \\+ lambda \\* beta must be > 0"):
        regularizers.DURA_regularizer(params)
    regularizers.DURA_regularizer({"alpha": 0.0})  # one weight 0 is fine
    regularizers.DURA_regularizer({"beta": 0.0})


# ---------------------------------------------------------------- refusals
@pytest.mark.parametrize("reg", [["DURA", None], [None, "DURA"], ["DURA", "DURA"], ["N3", "DURA"], ["DURA", "LP"]])
def test_list_forms_refused(reg):
    with pytest.raises(ValueError, match="DURA.*couples.*not in a list"):
        _model(reg=reg)


def test_list_form_of_an_instance_refused():
    from ampligraph_b200.latent_features import regularizers
    inst = regularizers.DURA_regularizer()
    with pytest.raises(ValueError, match="DURA"):
        _model(reg=[inst, inst])


@pytest.mark.parametrize("scoring", ["TransE", "RotatE"])
def test_translational_models_refused(scoring):
    with pytest.raises(NotImplementedError, match="DURA.*%s" % scoring):
        _model(scoring, loss="pairwise")


@pytest.mark.parametrize("scoring", ["DistMult", "ComplEx", "HolE"])
def test_tensor_factorisation_models_accepted(scoring):
    from ampligraph_b200.latent_features import regularizers
    m = _model(scoring)
    assert all(isinstance(r, regularizers.DURARegularizer) for r in m._regularizer)


def test_k_vs_all_refused():
    m = _model(loss="nll")
    with pytest.raises(NotImplementedError, match="DURA.*k_vs_all"):
        m.fit(X, epochs=1, k_vs_all="s,o")
    assert m.engine is None and m.data_indexer is True  # nothing was indexed or built


def test_several_gpus_refused(monkeypatch):
    from ampligraph_b200.latent_features import models
    monkeypatch.setattr(models.ScoringBasedEmbeddingModel, "_world", lambda self: 2)
    m = _model(loss="pairwise")
    for call in (lambda: m.fit(X, epochs=1), lambda: m.fit(X, epochs=1, one_vs_all="s,o"),
                 lambda: m.train_on_batch(X), lambda: m.train_on_batches([np.zeros((2, 3), np.int32)])):
        with pytest.raises(NotImplementedError, match="DURA.*single-GPU"):
            call()
    assert m.engine is None and m.data_indexer is True  # nothing was indexed or built


# ---------------------------------------------------------------- table rules and the engine config
@pytest.mark.parametrize("opt,hp,plain", [("adam", {}, (False, False)), ("adamax", {}, (True, True)),
                                          ("rmsprop", {"momentum": 0.9}, (True, True)),
                                          ("lazy_adam", {}, (True, True))])
def test_table_rules_with_dura(opt, hp, plain):
    """DURA keeps both tables' looked-up-rows rule wherever unregularised tables would have it."""
    from ampligraph_b200.latent_features import optimizers, regularizers
    params = [r.kernel_params() for r in regularizers.get_pair("DURA")]
    assert optimizers.table_rules(opt, hp, [not regularizers.is_per_occurrence(r) for r in params]) == plain
    assert optimizers.table_rules(opt, hp, [False, False]) == plain


class _FakeEngine:
    seen = {}

    def __init__(self, *a, **k):
        _FakeEngine.seen = dict(k)

    def __getattr__(self, name):
        return lambda *a, **k: None


@pytest.mark.parametrize("opt,want", [("adamax", (True, True)), ("adam", (False, False)), ("lazy_adam", (True, True))])
def test_build_engine_passes_dura_as_unregularised(monkeypatch, opt, want):
    """_build_engine: DURA goes to table_rules as unregularised and to the engine as the same {"kind": "DURA"} config
    for both tables, so the optimizer config carries no LP term."""
    from ampligraph_b200.latent_features import models
    monkeypatch.setattr(models, "KGEEngine", _FakeEngine)
    m = _model("DistMult", reg="DURA", optimizer=opt)
    m.max_ent_size, m.max_rel_size = 3, 2
    m._build_engine()
    cfg = {"kind": "DURA", "lambda": 1e-3, "alpha": 1.0, "beta": 1.0}
    assert _FakeEngine.seen["regularizer"] == [cfg, cfg]
    assert _FakeEngine.seen["lazy_tables"] == want


def test_engine_strips_dura_from_the_optimizer():
    """KGEEngine.set_optimizer keeps (w_n, w_p) = (lambda alpha, lambda beta) and gives the optimizer no regulariser;
    a DURA config on one table only is refused."""
    from ampligraph_b200 import _lib
    from ampligraph_b200.engine import KGEEngine
    eng = KGEEngine.__new__(KGEEngine)  # set_optimizer without a device: the slots and stamps are stubbed
    eng.ent_rows, eng.n_rel, eng.ld, eng.device = 2, 2, 4, "cpu"
    eng.h = None

    class Lib:
        def kge_set_row_stamps(self, *a):
            return 0
    eng.lib = Lib()
    cfg = {"kind": "DURA", "lambda": 0.1, "alpha": 0.5, "beta": 3.0}
    eng.set_optimizer("adam", {}, [cfg, dict(cfg)])
    assert eng.dura_weights == (0.1 * 0.5, 0.1 * 3.0)
    assert eng.n3_lambdas == {"ent": 0.0, "rel": 0.0}
    assert eng.opt_cfgs["ent"].reg_p == 0 and eng.opt_cfgs["rel"].reg_p == 0
    eng.set_optimizer("adam", {}, None)
    assert eng.dura_weights is None
    with pytest.raises(ValueError, match="DURA.*both"):
        eng.set_optimizer("adam", {}, [cfg, None])
    assert _lib.OPTIMIZERS["adam"] >= 0


# ---------------------------------------------------------------- grid
@pytest.mark.parametrize("name", ["DURA", "dura"])
def test_grid_takes_dura(name):
    """select_best_model_ranking's regularizer / regularizer_params grid keys build a DURA model unchanged."""
    from ampligraph_b200.evaluation import _build_model
    from ampligraph_b200.latent_features import regularizers
    m = _build_model("ComplEx", {"k": 8, "regularizer": name, "regularizer_params": {"lambda": 0.02, "beta": 0.5},
                                 "loss": "multiclass_nll"}, 2)
    r = m._regularizer[0]
    assert m._regularizer[1] is r and isinstance(r, regularizers.DURARegularizer)
    assert (r.lam, r.alpha, r.beta) == (0.02, 1.0, 0.5)


# ---------------------------------------------------------------- ABI
def test_abi_declares_and_exports_the_entry_point():
    from ampligraph_b200 import _lib
    if not os.path.exists(_lib.SO_PATH):
        _lib.build()
    lib = _lib.load()
    header = open(_lib.HEADER).read()
    assert re.search(r"\bkge_dura_step\s*\(", header)
    assert "kge_dura_step" in _lib.PROTOTYPES and getattr(lib, "kge_dura_step") is not None
    assert len(_lib.PROTOTYPES["kge_dura_step"][1]) == 12  # no workspace arguments
    assert _lib.ABI_VERSION == 2


# ---------------------------------------------------------------- oracle
def _numpy_loss(model, ent, rel, triples, w_n, w_p):
    total = 0.0
    for h, r, t in triples:
        rows = [ent[h], rel[r], ent[t]]
        if model in dura_oracle.TWO_HALVES:
            k = ent.shape[1] // 2
            hc, rc, tc = (x[:k] + 1j * x[k:] for x in rows)
            total += w_n * (np.sum(np.abs(hc) ** 2) + np.sum(np.abs(tc) ** 2))
            total += w_p * (np.sum(np.abs(hc * rc) ** 2) + np.sum(np.abs(tc * np.conj(rc)) ** 2))
        else:
            hc, rc, tc = rows
            total += w_n * (np.sum(hc ** 2) + np.sum(tc ** 2)) + w_p * (np.sum((hc * rc) ** 2) + np.sum((tc * rc) ** 2))
    return total


TRIPLES = np.array([[0, 1, 3], [2, 0, 2], [0, 1, 3], [4, 2, 0], [1, 1, 1]])  # a repeated positive and two self-loops


@pytest.mark.parametrize("model", ["DistMult", "ComplEx", "HolE"])
@pytest.mark.parametrize("w", [(0.5, 0.25), (0.0, 0.75), (0.375, 0.0)])
def test_oracle_vs_numpy(model, w):
    """Loss (the paper's complex form) and central-difference gradients against a numpy restatement; rows repeat
    within the batch, self-loops, and one component exactly 0."""
    rng = np.random.default_rng(5)
    E, R, K = 5, 3, 6
    ent, rel = rng.uniform(-1, 1, (E, K)), rng.uniform(-1, 1, (R, K))
    ent[2, 1] = 0.0
    loss, g_ent, g_rel = dura_oracle.loss_and_grads(model, ent, rel, TRIPLES, *w)
    assert loss == pytest.approx(_numpy_loss(model, ent, rel, TRIPLES, *w), rel=1e-12)
    for table, grad in ((ent, g_ent), (rel, g_rel)):
        num = np.zeros_like(table)
        for idx in np.ndindex(*table.shape):
            h = 1e-6
            table[idx] += h
            up = _numpy_loss(model, ent, rel, TRIPLES, *w)
            table[idx] -= 2 * h
            down = _numpy_loss(model, ent, rel, TRIPLES, *w)
            table[idx] += h
            num[idx] = (up - down) / (2 * h)
        assert np.allclose(grad, num, rtol=1e-6, atol=1e-8), np.abs(grad - num).max()
    if w[1] == 0.0:
        assert not g_rel.any()


@pytest.mark.parametrize("model", ["DistMult", "ComplEx"])
def test_oracle_closed_form_per_row(model):
    """Per occurrence equals per row: g_x = 2 x sum (w_n + w_p m_r) over x's occurrences as h or t (a self-loop counts
    twice), g_r = 2 w_p r sum (m_h + m_t)."""
    rng = np.random.default_rng(9)
    ent, rel = rng.uniform(-1, 1, (4, 8)), rng.uniform(-1, 1, (2, 8))
    t = np.array([[0, 0, 0], [1, 1, 2], [0, 1, 3], [3, 0, 0], [1, 1, 2]])
    _, g_ent, g_rel = dura_oracle.loss_and_grads(model, ent, rel, t, 0.125, 0.5)
    ce, cr = dura_oracle.occurrences(t, 4, 2)
    assert ce.tolist() == [4, 2, 2, 2] and cr.tolist() == [2, 3]
    ge, gr = dura_oracle.closed_form(model, ent, rel, t, 0.125, 0.5)
    assert np.allclose(ge, g_ent, rtol=1e-13, atol=0) and np.allclose(gr, g_rel, rtol=1e-13, atol=0)
    if model == "DistMult":  # row 2 occurs twice, as t of (1, 1, 2): 2 x (2 (0.125 + 0.5 m_r1))
        assert np.allclose(g_ent[2], 2 * ent[2] * 2 * (0.125 + 0.5 * rel[1] ** 2), rtol=1e-13)


def test_oracle_bound_catches_a_lost_occurrence():
    """The per-element bound is tight enough that one occurrence more or less of a cold row falls outside it."""
    rng = np.random.default_rng(3)
    E, R, K, B = 200, 7, 16, 300
    ent, rel = rng.uniform(-0.3, 0.3, (E, K)), rng.uniform(-0.3, 0.3, (R, K))
    t = np.stack([rng.integers(0, E, B), rng.integers(0, R, B), rng.integers(0, E, B)], 1)
    lb, be, br = dura_oracle.bound("ComplEx", ent, rel, t, 1e-3, 2e-3)
    _, ge, gr = dura_oracle.loss_and_grads("ComplEx", ent, rel, t, 1e-3, 2e-3)
    _, ge1, gr1 = dura_oracle.loss_and_grads("ComplEx", ent, rel, t[1:], 1e-3, 2e-3)  # positive 0 lost
    _, ge2, gr2 = dura_oracle.loss_and_grads("ComplEx", ent, rel, np.concatenate([t, t[:1]]), 1e-3, 2e-3)  # doubled
    ce, _ = dura_oracle.occurrences(t, E, R)
    cold = t[0, 0] if ce[t[0, 0]] <= 2 else t[0, 2]
    for g in (ge1, ge2):
        assert (np.abs(g[cold] - ge[cold]) > be[cold]).any()
    for g in (gr1, gr2):
        assert (np.abs(g[t[0, 1]] - gr[t[0, 1]]) > br[t[0, 1]]).any()
    assert np.all(be >= 0) and lb > 0
