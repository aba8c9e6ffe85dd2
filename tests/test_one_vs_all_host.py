"""CPU tests (no GPU) of 1vsAll training: the refusals of fit(one_vs_all=...), the C-ABI's two entry points, the
workspace-size formula and the float64 oracle (tests/one_vs_all_oracle.py) against a plain numpy restatement."""
import os
import re

import numpy as np
import pytest

import one_vs_all_oracle

X = np.array([["a", "r", "b"], ["b", "r", "c"], ["c", "q", "a"]])


def _model(scoring="ComplEx", loss="multiclass_nll"):
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    m = ScoringBasedEmbeddingModel(eta=2, k=4, scoring_type=scoring)
    m.compile(optimizer="adam", loss=loss)
    return m


@pytest.mark.parametrize("bad", ["so", "o,s", "", "p", 1, ("s", "o")])
def test_bad_sides_refused(bad):
    with pytest.raises(ValueError, match="one_vs_all"):
        _model().fit(X, epochs=1, one_vs_all=bad)


@pytest.mark.parametrize("scoring", ["TransE", "RotatE"])
def test_distance_models_refused(scoring):
    with pytest.raises(NotImplementedError, match="DistMult, ComplEx and HolE"):
        _model(scoring).fit(X, epochs=1, one_vs_all="s,o")


@pytest.mark.parametrize("loss", ["pairwise", "nll", "absolute_margin", "self_adversarial", lambda sp, sn: sp])
def test_other_losses_refused(loss):
    with pytest.raises(ValueError, match="multiclass_nll"):
        _model(loss=loss).fit(X, epochs=1, one_vs_all="o")


def test_focuse_and_multi_gpu_refused():
    with pytest.raises(NotImplementedError, match="focusE"):
        _model().fit(np.concatenate([X, [["1"], ["2"], ["3"]]], 1), epochs=1, focusE=True, one_vs_all="s,o")
    m = _model()
    m._world = lambda: 2  # as under torchrun with two ranks
    with pytest.raises(NotImplementedError, match="single-GPU"):
        m.fit(X, epochs=1, one_vs_all="s")


def test_abi_declares_and_exports_the_entry_points():
    from ampligraph_b200 import _lib
    if not os.path.exists(_lib.SO_PATH):
        _lib.build()
    lib = _lib.load()
    header = open(_lib.HEADER).read()
    for name in ("kge_one_vs_all_step", "kge_one_vs_all_workspace_bytes"):
        assert re.search(r"\b%s\s*\(" % name, header), name
        assert name in _lib.PROTOTYPES and getattr(lib, name) is not None
    assert re.search(r"KGE_ONE_VS_ALL_S\s*=\s*1\s*,\s*KGE_ONE_VS_ALL_O\s*=\s*2", header)
    assert _lib.ONE_VS_ALL_SIDES == {"s": 1, "o": 2, "s,o": 3}
    assert lib.kge_one_vs_all_workspace_bytes(None, 10) == 0  # null handle


def test_workspace_formula():
    from ampligraph_b200.engine import one_vs_all_splits, one_vs_all_workspace_bytes
    # splits: ~264 CTAs over the query tiles, at most 64, at most one per 32-entity tile
    assert one_vs_all_splits(1000, 14541) == 9       # 32 query tiles
    assert one_vs_all_splits(4096, 14541) == 3       # 128 query tiles
    assert one_vs_all_splits(10, 1_000_000) == 64    # capped
    assert one_vs_all_splits(10, 40) == 2            # two entity tiles
    assert one_vs_all_splits(100_000, 50) == 1
    assert one_vs_all_workspace_bytes(0, 100, 8) == 0
    # B = 3, ld = 8, one split (one entity tile): 2 * 96 + 16 + 2 * 16 + 3 * 16 + 96
    assert one_vs_all_workspace_bytes(3, 20, 8) == 2 * 96 + 16 + 2 * 16 + 3 * 16 + 96
    B, ld = 1000, 400
    ns = one_vs_all_splits(B, 14541)
    assert one_vs_all_workspace_bytes(B, 14541, ld) == (2 + ns) * 4 * B * ld + (4 + 2 * ns) * 4 * B


def _numpy_scores(model, ent, rel, s, p, o):
    """f(s, p, o) of the reference's scoring layers (DistMult.py:48, ComplEx.py:52-62, HolE.py:45), one triple."""
    K = ent.shape[1]
    if model == "DistMult":
        return float(np.sum(ent[s] * rel[p] * ent[o]))
    h = K // 2
    sr, si, pr, pi, orr, oi = ent[s, :h], ent[s, h:], rel[p, :h], rel[p, h:], ent[o, :h], ent[o, h:]
    sc = float(np.sum(sr * (pr * orr + pi * oi) + si * (pr * oi - pi * orr)))
    return sc * 2.0 / (K / 2.0) if model == "HolE" else sc


def _numpy_loss(model, ent, rel, triples, sides, reduction):
    n = ent.shape[0]
    total = 0.0
    for s, p, o in triples:
        for side in sides.split(","):
            lg = np.array([_numpy_scores(model, ent, rel, e, p, o) if side == "s" else _numpy_scores(model, ent, rel, s, p, e)
                           for e in range(n)])
            lg = np.clip(lg, -75.0, 75.0)
            t = s if side == "s" else o
            if reduction == "sum":
                total += np.log(np.sum(np.exp(lg))) - lg[t]
            else:
                neg = np.delete(np.exp(lg), t)
                total += -np.log(np.exp(lg[t]) / (neg.mean() + np.exp(lg[t])))
    return total


@pytest.mark.parametrize("model", ["DistMult", "ComplEx", "HolE"])
@pytest.mark.parametrize("sides", ["s,o", "o", "s"])
@pytest.mark.parametrize("reduction", ["sum", "mean"])
def test_oracle_vs_numpy(model, sides, reduction):
    """Loss and central-difference gradients of the numpy restatement against the oracle, both float64; one logit is
    pushed past the clip so that its zero gradient is covered."""
    rng = np.random.default_rng(3)
    E, R, K = 5, 2, 4
    ent, rel = rng.uniform(-1, 1, (E, K)), rng.uniform(-1, 1, (R, K))
    triples = np.array([[0, 1, 3], [2, 0, 2], [4, 1, 0]])
    if model == "DistMult":
        ent[1] *= 40.0
        rel[1] *= 40.0  # f(0, 1, 1) and f(1, 1, 3) leave [-75, 75]
    for matmul in (False, True):
        loss, g_ent, g_rel = one_vs_all_oracle.loss_and_grads(model, ent, rel, triples, sides, reduction, matmul=matmul)
        assert loss == pytest.approx(_numpy_loss(model, ent, rel, triples, sides, reduction), rel=1e-12)
        for table, grad in ((ent, g_ent), (rel, g_rel)):
            num = np.zeros_like(table)
            for idx in np.ndindex(*table.shape):
                h = 1e-6
                table[idx] += h
                up = _numpy_loss(model, ent, rel, triples, sides, reduction)
                table[idx] -= 2 * h
                down = _numpy_loss(model, ent, rel, triples, sides, reduction)
                table[idx] += h
                num[idx] = (up - down) / (2 * h)
            assert np.allclose(grad, num, rtol=1e-5, atol=1e-6), (matmul, np.abs(grad - num).max())
