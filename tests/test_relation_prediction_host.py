"""CPU tests (no GPU, but for one check against a live handle) of relation prediction as an auxiliary 1vsAll objective:
the refusals of fit(relation_prediction_weight=...), the C-ABI's two entry points, the workspace-size formula and the float64 oracle
(tests/relation_prediction_oracle.py) against a plain numpy restatement."""
import os
import re

import numpy as np
import pytest

import relation_prediction_oracle

X = np.array([["a", "r", "b"], ["b", "r", "c"], ["c", "q", "a"]])


def _model(scoring="ComplEx", loss="multiclass_nll"):
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    m = ScoringBasedEmbeddingModel(eta=2, k=4, scoring_type=scoring)
    m.compile(optimizer="adam", loss=loss)
    return m


@pytest.mark.parametrize("bad", [True, False, float("nan"), float("inf"), -float("inf"), -0.5, "1", None])
def test_bad_weight_refused(bad):
    with pytest.raises(ValueError, match="relation_prediction_weight"):
        _model().fit(X, epochs=1, one_vs_all="s,o", relation_prediction_weight=bad)


def test_weight_needs_one_vs_all():
    with pytest.raises(ValueError, match="one_vs_all"):
        _model().fit(X, epochs=1, relation_prediction_weight=1.0)
    with pytest.raises(ValueError, match="k_vs_all"):
        _model(loss="nll").fit(X, epochs=1, k_vs_all="s,o", relation_prediction_weight=1.0)


def test_one_relation_refused():
    with pytest.raises(ValueError, match="two relations"):
        _model().fit(X[:2], epochs=1, one_vs_all="s,o", relation_prediction_weight=0.5)


def test_one_vs_all_refusals_still_apply():
    with pytest.raises(NotImplementedError, match="DistMult, ComplEx and HolE"):
        _model("TransE").fit(X, epochs=1, one_vs_all="s,o", relation_prediction_weight=1.0)
    with pytest.raises(ValueError, match="multiclass_nll"):
        _model(loss="pairwise").fit(X, epochs=1, one_vs_all="s,o", relation_prediction_weight=1.0)


def test_abi_declares_and_exports_the_entry_points():
    from ampligraph_b200 import _lib
    if not os.path.exists(_lib.SO_PATH):
        _lib.build()
    lib = _lib.load()
    header = open(_lib.HEADER).read()
    for name in ("kge_one_vs_all_relation_step", "kge_one_vs_all_relation_workspace_bytes"):
        assert re.search(r"\b%s\s*\(" % name, header), name
        assert name in _lib.PROTOTYPES and getattr(lib, name) is not None
    assert lib.kge_one_vs_all_relation_workspace_bytes(None, 10) == 0  # null handle


def test_workspace_formula():
    from ampligraph_b200.engine import one_vs_all_relation_workspace_bytes, one_vs_all_splits
    # dX splits the query tiles of each 32-relation tile with the same rule, roles swapped
    assert one_vs_all_splits(237, 1000) == 32    # 8 relation tiles, 32 query tiles
    assert one_vs_all_splits(237, 4096) == 33    # 8 relation tiles: ceil(264 / 8)
    assert one_vs_all_splits(237, 20) == 1       # one query tile: dX adds to g_rel directly
    assert one_vs_all_relation_workspace_bytes(0, 237, 400) == 0
    # B = 3, n_rel = 5, ld = 8: one split each way: 96 + 2 * 16 + 3 * 16 + 96
    assert one_vs_all_relation_workspace_bytes(3, 5, 8) == 96 + 2 * 16 + 3 * 16 + 96
    B, R, ld = 1000, 237, 400
    ns, xs = one_vs_all_splits(B, R), one_vs_all_splits(R, B)
    assert ns == 8
    assert one_vs_all_relation_workspace_bytes(B, R, ld) == (1 + ns) * 4 * B * ld + (3 + 2 * ns) * 4 * B + xs * 4 * R * ld


@pytest.mark.gpu
@pytest.mark.gpu
def test_workspace_formula_matches_the_library():
    """A handle needs a device."""
    from ampligraph_b200 import _lib
    from ampligraph_b200.engine import KGEEngine, one_vs_all_relation_workspace_bytes
    lib = _lib.load()
    for R, k in ((2, 4), (40, 10), (237, 200)):
        eng = KGEEngine("ComplEx", k, 1, 100, R, loss="multiclass_nll")
        for B in (0, 1, 31, 50, 1000, 4096):
            assert lib.kge_one_vs_all_relation_workspace_bytes(eng.h, B) == one_vs_all_relation_workspace_bytes(B, R, eng.ld)
        eng.close()


def _numpy_score(model, ent, rel, s, p, o):
    """f(s, p, o) of the reference's scoring layers (DistMult.py:48, ComplEx.py:52-62, HolE.py:45), one triple."""
    K = ent.shape[1]
    if model == "DistMult":
        return float(np.sum(ent[s] * rel[p] * ent[o]))
    h = K // 2
    sr, si, pr, pi, orr, oi = ent[s, :h], ent[s, h:], rel[p, :h], rel[p, h:], ent[o, :h], ent[o, h:]
    sc = float(np.sum(sr * (pr * orr + pi * oi) + si * (pr * oi - pi * orr)))
    return sc * 2.0 / (K / 2.0) if model == "HolE" else sc


def _numpy_loss(model, ent, rel, triples, weight, reduction):
    total = 0.0
    for s, p, o in triples:
        lg = np.clip([_numpy_score(model, ent, rel, s, r, o) for r in range(rel.shape[0])], -75.0, 75.0)
        if reduction == "sum":
            total += np.log(np.sum(np.exp(lg))) - lg[p]
        else:
            neg = np.delete(np.exp(lg), p)
            total += -np.log(np.exp(lg[p]) / (neg.mean() + np.exp(lg[p])))
    return weight * total


@pytest.mark.parametrize("model", ["DistMult", "ComplEx", "HolE"])
@pytest.mark.parametrize("reduction", ["sum", "mean"])
def test_oracle_vs_numpy(model, reduction):
    """Loss and central-difference gradients of the numpy restatement against the oracle, both float64, in both forms
    of the logits; one logit is pushed past the clip so that its zero gradient is covered."""
    rng = np.random.default_rng(3)
    E, R, K = 5, 4, 4
    ent, rel = rng.uniform(-1, 1, (E, K)), rng.uniform(-1, 1, (R, K))
    triples = np.array([[0, 1, 3], [2, 0, 2], [4, 3, 0], [1, 2, 1]])
    ent[1] *= 40.0
    rel[2] *= 40.0  # f(1, 2, 1) leaves [-75, 75]
    assert abs(_numpy_score(model, ent, rel, 1, 2, 1)) > 75.0
    weight = 0.75
    for matmul in (False, True):
        loss, g_ent, g_rel = relation_prediction_oracle.loss_and_grads(model, ent, rel, triples, weight, reduction,
                                                                        matmul=matmul)
        assert loss == pytest.approx(_numpy_loss(model, ent, rel, triples, weight, reduction), rel=1e-12)
        for table, grad in ((ent, g_ent), (rel, g_rel)):
            num = np.zeros_like(table)
            for idx in np.ndindex(*table.shape):
                h = 1e-6
                table[idx] += h
                up = _numpy_loss(model, ent, rel, triples, weight, reduction)
                table[idx] -= 2 * h
                down = _numpy_loss(model, ent, rel, triples, weight, reduction)
                table[idx] += h
                num[idx] = (up - down) / (2 * h)
            assert np.allclose(grad, num, rtol=1e-5, atol=1e-6), (matmul, np.abs(grad - num).max())


def test_oracle_adds_the_entity_sides():
    """With sides, the oracle is the 1vsAll oracle's L_s + L_o plus weight * L_p."""
    import one_vs_all_oracle
    rng = np.random.default_rng(7)
    ent, rel = rng.uniform(-1, 1, (6, 8)), rng.uniform(-1, 1, (3, 8))
    t = np.array([[0, 1, 3], [2, 0, 5], [4, 2, 0]])
    both = relation_prediction_oracle.loss_and_grads("ComplEx", ent, rel, t, 2.0, "sum", sides="s,o")
    ent_only = one_vs_all_oracle.loss_and_grads("ComplEx", ent, rel, t, "s,o", "sum")
    rel_only = relation_prediction_oracle.loss_and_grads("ComplEx", ent, rel, t, 2.0, "sum")
    assert both[0] == pytest.approx(ent_only[0] + rel_only[0], rel=1e-12)
    for i in (1, 2):
        assert np.allclose(both[i], ent_only[i] + rel_only[i], rtol=1e-12, atol=1e-12)
