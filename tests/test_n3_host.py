"""CPU tests of the N3 regulariser: the registry, the optimizer's per-table rule with N3, the refusals (before anything
is indexed or trained), the C-ABI's two entry points and the workspace formula, select_best_model_ranking's grid, and the
float64 oracle (tests/n3_oracle.py) against a numpy restatement and central differences."""
import os
import re

import numpy as np
import pytest

import n3_oracle

X = np.array([["a", "r", "b"], ["b", "r", "c"], ["c", "q", "a"]])


def _model(scoring="ComplEx", loss="multiclass_nll", reg="N3", optimizer="adam"):
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    m = ScoringBasedEmbeddingModel(eta=2, k=4, scoring_type=scoring)
    m.compile(optimizer=optimizer, loss=loss, entity_relation_regularizer=reg)
    return m


# ---------------------------------------------------------------- registry
def test_registry_names_and_default_lambda():
    from ampligraph_b200.latent_features import regularizers
    for name in ("N3", "n3"):
        r = regularizers.get(name)
        assert isinstance(r, regularizers.N3Regularizer) and r.__name__ == "N3" and r.lam == 1e-3
        assert r.kernel_params() == {"kind": "N3", "lambda": 1e-3}
        assert regularizers.is_n3(r.kernel_params())
    assert regularizers.get("N3", {"lambda": 0.05}).lam == 0.05
    inst = regularizers.N3_regularizer({"lambda": 0.25})
    assert regularizers.get(inst) is inst
    assert regularizers.get_pair(inst) == [inst, inst]
    pair = regularizers.get_pair(["N3", None], {"lambda": 0.5})
    assert isinstance(pair[0], regularizers.N3Regularizer) and pair[0].lam == 0.5 and pair[1] is None
    pair = regularizers.get_pair([None, "n3"])
    assert pair[0] is None and isinstance(pair[1], regularizers.N3Regularizer)
    mixed = regularizers.get_pair(["LP", "N3"], {"p": 3, "lambda": 0.1})
    assert isinstance(mixed[0], regularizers.LPRegularizer) and mixed[0].p == 3 and mixed[1].lam == 0.1
    assert not regularizers.is_n3(mixed[0].kernel_params()) and not regularizers.is_n3(None)


def test_registry_unchanged_for_other_names():
    from ampligraph_b200.latent_features import regularizers
    assert regularizers.get("l3").p == 3 and regularizers.get("LP").lam == 1e-5
    for bad in ("N4", "nuclear", "lp", {"class_name": "N3"}):
        with pytest.raises(ValueError, match=re.escape("Could not interpret regularizer identifier: %r" % (bad,))):
            regularizers.get(bad)


@pytest.mark.parametrize("bad", [-1.0, float("nan"), float("inf")])
def test_bad_lambda_refused(bad):
    from ampligraph_b200.latent_features import regularizers
    with pytest.raises(ValueError, match="N3"):
        regularizers.N3_regularizer({"lambda": bad})


# ---------------------------------------------------------------- table rules
@pytest.mark.parametrize("opt,hp,plain", [("adam", {}, (False, False)), ("adamax", {}, (True, True)),
                                          ("rmsprop", {"momentum": 0.9}, (True, True)),
                                          ("lazy_adam", {}, (True, True))])
@pytest.mark.parametrize("reg", [["N3", "N3"], ["N3", None], [None, "N3"], ["LP", "N3"], ["N3", "LP"]])
def test_table_rules_with_n3(opt, hp, plain, reg):
    """N3 keeps a table's looked-up-rows rule wherever an unregularised table would have it; an LP table stays dense
    (lazy_ asks for the looked-up rows on both tables whatever the regulariser)."""
    from ampligraph_b200.latent_features import optimizers, regularizers
    regs = regularizers.get_pair(reg)
    params = [r.kernel_params() if r is not None else None for r in regs]
    got = optimizers.table_rules(opt, hp, [r is not None and not regularizers.is_n3(r) for r in params])
    lazy_prefix = opt.startswith("lazy_")
    want = tuple(p if (lazy_prefix or not isinstance(r, regularizers.LPRegularizer)) else False
                 for p, r in zip(plain, regs))
    assert got == want


def test_build_engine_passes_n3_as_unregularised(monkeypatch):
    """_build_engine: the N3 table goes to table_rules as unregularised and to the engine as {"kind": "N3"}, so the
    optimizer config carries no LP term for it."""
    from ampligraph_b200.latent_features import models
    seen = {}

    class Fake:
        def __init__(self, *a, **k):
            seen.update(k)

        def __getattr__(self, name):
            return lambda *a, **k: None

    monkeypatch.setattr(models, "KGEEngine", Fake)
    m = _model("DistMult", reg=["N3", "LP"], optimizer="adamax")
    m.max_ent_size, m.max_rel_size = 3, 2
    m._build_engine()
    assert seen["regularizer"][0] == {"kind": "N3", "lambda": 1e-3}
    assert seen["regularizer"][1]["p"] == 2
    assert seen["lazy_tables"] == (True, False)


# ---------------------------------------------------------------- refusals
def test_rotate_relation_n3_refused():
    with pytest.raises(NotImplementedError, match="N3"):
        _model("RotatE", loss="pairwise", reg="N3")
    with pytest.raises(NotImplementedError, match="N3"):
        _model("RotatE", loss="pairwise", reg=[None, "N3"])
    _model("RotatE", loss="pairwise", reg=["N3", None])  # the entity table is fine


def test_k_vs_all_refused():
    with pytest.raises(NotImplementedError, match="N3.*k_vs_all"):
        _model(loss="nll").fit(X, epochs=1, k_vs_all="s,o")


def test_several_gpus_refused(monkeypatch):
    from ampligraph_b200.latent_features import models
    monkeypatch.setattr(models.ScoringBasedEmbeddingModel, "_world", lambda self: 2)
    m = _model(loss="pairwise")
    for call in (lambda: m.fit(X, epochs=1), lambda: m.train_on_batch(X),
                 lambda: m.train_on_batches([np.zeros((2, 3), np.int32)])):
        with pytest.raises(NotImplementedError, match="N3.*single-GPU"):
            call()
    assert m.engine is None and m.data_indexer is True  # nothing was indexed or built


def test_grid_takes_n3():
    """select_best_model_ranking's regularizer / regularizer_params grid keys build an N3 model unchanged."""
    from ampligraph_b200.evaluation import _build_model
    from ampligraph_b200.latent_features import regularizers
    m = _build_model("ComplEx", {"k": 8, "regularizer": "N3", "regularizer_params": {"lambda": 0.02},
                                 "loss": "multiclass_nll"}, 2)
    assert all(isinstance(r, regularizers.N3Regularizer) and r.lam == 0.02 for r in m._regularizer)


# ---------------------------------------------------------------- ABI
def test_abi_declares_and_exports_the_entry_points():
    from ampligraph_b200 import _lib
    if not os.path.exists(_lib.SO_PATH):
        _lib.build()
    lib = _lib.load()
    header = open(_lib.HEADER).read()
    for name in ("kge_n3_step", "kge_n3_workspace_bytes"):
        assert re.search(r"\b%s\s*\(" % name, header), name
        assert name in _lib.PROTOTYPES and getattr(lib, name) is not None
    assert lib.kge_n3_workspace_bytes(None) == 0  # null handle
    assert _lib.ABI_VERSION == 2


def test_workspace_formula():
    from ampligraph_b200.engine import KGEEngine
    eng = KGEEngine.__new__(KGEEngine)  # the property reads n_ent and n_rel only
    for E, R, want in ((1, 1, 16), (2, 2, 16), (3, 2, 32), (14541, 237, 59120), (10 ** 6, 1000, 4004000)):
        eng.n_ent, eng.n_rel = E, R
        assert eng.n3_workspace_bytes == want == (4 * (E + R) + 15) // 16 * 16


# ---------------------------------------------------------------- oracle
def _numpy_loss(model, ent, rel, triples, le, lr):
    total = 0.0
    for s, p, o in triples:
        for lam, row in ((le, ent[s]), (le, ent[o]), (lr, rel[p])):
            if model in n3_oracle.TWO_HALVES:
                h = row.shape[0] // 2
                total += lam * np.sum(np.sqrt(row[:h] ** 2 + row[h:] ** 2) ** 3)
            else:
                total += lam * np.sum(np.abs(row) ** 3)
    return total


@pytest.mark.parametrize("model", ["TransE", "DistMult", "ComplEx", "HolE", "RotatE"])
def test_oracle_vs_numpy(model):
    """Loss and central-difference gradients against a numpy restatement; rows repeat within the batch, an entity is
    both s and o of one positive, and one row component is exactly 0."""
    rng = np.random.default_rng(5)
    E, R, K = 5, 3, 6
    ent, rel = rng.uniform(-1, 1, (E, K)), rng.uniform(-1, 1, (R, K))
    ent[2, 1] = 0.0
    triples = np.array([[0, 1, 3], [2, 0, 2], [0, 1, 3], [4, 2, 0], [1, 1, 1]])
    le, lr = 0.5, 0.25 if model != "RotatE" else 0.0
    loss, g_ent, g_rel = n3_oracle.loss_and_grads(model, ent, rel, triples, le, lr)
    assert loss == pytest.approx(_numpy_loss(model, ent, rel, triples, le, lr), rel=1e-12)
    for table, grad in ((ent, g_ent), (rel, g_rel)):
        num = np.zeros_like(table)
        for idx in np.ndindex(*table.shape):
            h = 1e-6
            table[idx] += h
            up = _numpy_loss(model, ent, rel, triples, le, lr)
            table[idx] -= 2 * h
            down = _numpy_loss(model, ent, rel, triples, le, lr)
            table[idx] += h
            num[idx] = (up - down) / (2 * h)
        assert np.allclose(grad, num, rtol=1e-6, atol=1e-8), np.abs(grad - num).max()
    if lr == 0.0:
        assert not g_rel.any()


def test_oracle_closed_form_per_row():
    """Per occurrence equals per row: g = c * 3 lambda |z| z, the form the kernel uses."""
    rng = np.random.default_rng(9)
    ent, rel = rng.uniform(-1, 1, (4, 8)), rng.uniform(-1, 1, (2, 8))
    t = np.array([[0, 0, 0], [1, 1, 2], [0, 1, 3], [3, 0, 0]])
    _, g_ent, g_rel = n3_oracle.loss_and_grads("ComplEx", ent, rel, t, 0.125, 0.5)
    ce, cr = n3_oracle.counts(t, 4, 2)
    assert ce.tolist() == [4, 1, 1, 2] and cr.tolist() == [2, 2]
    for table, c, lam, g in ((ent, ce, 0.125, g_ent), (rel, cr, 0.5, g_rel)):
        m = np.sqrt(table[:, :4] ** 2 + table[:, 4:] ** 2)
        assert np.allclose(g, 3 * lam * c[:, None] * np.concatenate([m, m], 1) * table, rtol=1e-13, atol=0)
