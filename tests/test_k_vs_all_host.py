"""CPU tests (no GPU) of KvsAll training: the refusals of fit(k_vs_all=...), the C-ABI's two entry points, the
workspace-size formula, the query grouping and epoch schedule against plain dict loops, and the float64 oracle
(tests/k_vs_all_oracle.py) against a numpy restatement and the reference's nll."""
import os
import re

import numpy as np
import pytest
import torch

import k_vs_all_oracle
from ampligraph_b200.datasets import FilterIndex, k_vs_all_queries, k_vs_all_steps
from oracle import ref_step

X = np.array([["a", "r", "b"], ["b", "r", "c"], ["c", "q", "a"]])


def _model(scoring="ComplEx", loss="nll"):
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    m = ScoringBasedEmbeddingModel(eta=2, k=4, scoring_type=scoring)
    m.compile(optimizer="adam", loss=loss)
    return m


@pytest.mark.parametrize("bad", ["so", "o,s", "", "p", 1, ("s", "o")])
def test_bad_sides_refused(bad):
    with pytest.raises(ValueError, match="k_vs_all"):
        _model().fit(X, epochs=1, k_vs_all=bad)


def test_with_one_vs_all_refused():
    with pytest.raises(ValueError, match="one_vs_all"):
        _model().fit(X, epochs=1, k_vs_all="o", one_vs_all="o")


@pytest.mark.parametrize("scoring", ["TransE", "RotatE"])
def test_distance_models_refused(scoring):
    with pytest.raises(NotImplementedError, match="DistMult, ComplEx and HolE"):
        _model(scoring).fit(X, epochs=1, k_vs_all="s,o")


@pytest.mark.parametrize("loss", ["pairwise", "multiclass_nll", "absolute_margin", "self_adversarial",
                                  lambda sp, sn: sp])
def test_other_losses_refused(loss):
    with pytest.raises(ValueError, match="'nll'"):
        _model(loss=loss).fit(X, epochs=1, k_vs_all="o")


@pytest.mark.parametrize("eps", [-0.1, 1.0, 1.5, float("nan"), float("inf"), "0.1", None, True])
def test_bad_label_smoothing_refused(eps):
    with pytest.raises(ValueError, match="label_smoothing"):
        _model().fit(X, epochs=1, k_vs_all="s,o", label_smoothing=eps)


def test_label_smoothing_without_k_vs_all_refused():
    with pytest.raises(ValueError, match="label_smoothing"):
        _model().fit(X, epochs=1, label_smoothing=0.1)
    with pytest.raises(ValueError, match="label_smoothing"):
        _model(loss="multiclass_nll").fit(X, epochs=1, one_vs_all="o", label_smoothing=0.1)


def test_focuse_and_multi_gpu_refused():
    with pytest.raises(NotImplementedError, match="focusE"):
        _model().fit(np.concatenate([X, [["1"], ["2"], ["3"]]], 1), epochs=1, focusE=True, k_vs_all="s,o")
    m = _model()
    m._world = lambda: 2  # as under torchrun with two ranks
    with pytest.raises(NotImplementedError, match="single-GPU"):
        m.fit(X, epochs=1, k_vs_all="s")


def test_abi_declares_and_exports_the_entry_points():
    from ampligraph_b200 import _lib
    if not os.path.exists(_lib.SO_PATH):
        _lib.build()
    lib = _lib.load()
    header = open(_lib.HEADER).read()
    for name in ("kge_k_vs_all_step", "kge_k_vs_all_workspace_bytes"):
        assert re.search(r"\b%s\s*\(" % name, header), name
        assert name in _lib.PROTOTYPES and getattr(lib, name) is not None
    assert lib.kge_k_vs_all_workspace_bytes(None, 10) == 0  # null handle


def test_workspace_formula():
    from ampligraph_b200.engine import k_vs_all_workspace_bytes, one_vs_all_splits
    assert k_vs_all_workspace_bytes(0, 100, 8) == 0
    # B = 3, ld = 8, one split (one entity tile): 2 * 96 + 16 + 96
    assert k_vs_all_workspace_bytes(3, 20, 8) == 2 * 96 + 16 + 96
    for B, n_ent, ld in ((1000, 14541, 400), (256, 14541, 400), (4096, 50, 12), (37, 1_000_000, 4)):
        ns = one_vs_all_splits(B, n_ent)
        assert k_vs_all_workspace_bytes(B, n_ent, ld) == (2 + ns) * 4 * B * ld + (4 * B + 15) // 16 * 16


def _random_triples(rng, n, E, R):
    t = np.stack([rng.integers(0, E, n), rng.integers(0, R, n), rng.integers(0, E, n)], 1)
    return np.concatenate([t, t[: n // 5]])  # repeated triples count once


@pytest.mark.parametrize("side", ["o", "s"])
def test_grouping_matches_dict_loop(side):
    rng = np.random.default_rng(7)
    E, R = 40, 3
    t = _random_triples(rng, 400, E, R)
    queries, off, ids = k_vs_all_queries(FilterIndex(t, E), t, side)
    keys, labels = k_vs_all_oracle.group(t, side)
    assert queries.dtype == np.int32 and off.dtype == np.int64 and ids.dtype == np.int32
    assert len(queries) == len(keys) and off[0] == 0 and off[-1] == len(ids)
    assert (queries == k_vs_all_oracle.query_rows(keys, labels, side)).all()  # first appearance, first label
    for i, lab in enumerate(labels):
        got = ids[off[i]:off[i + 1]].tolist()
        assert got == lab and got == sorted(set(got)), i
    assert sum(len(lab) for lab in labels) == len(np.unique(t, axis=0))  # every distinct triple is one label


@pytest.mark.parametrize("n_o,n_s,bs", [(10, 0, 3), (0, 7, 7), (0, 8, 3), (13, 29, 5), (100, 3, 10), (5, 5, 1),
                                        (1, 1, 1000), (333, 444, 64)])
def test_steps_cover_every_query_once(n_o, n_s, bs):
    got = k_vs_all_steps(n_o, n_s, bs)
    assert got == k_vs_all_oracle.steps(n_o, n_s, bs)
    for k, n in ((0, n_o), (1, n_s)):
        covered = [i for step in got for i in range(*step[k])]
        assert covered == list(range(n))
    assert all((o[1] - o[0]) + (s[1] - s[0]) <= bs + 1 for o, s in got)
    if n_o and n_s:
        assert len(got) == -(-(n_o + n_s) // bs)
    else:
        assert all((o[1] - o[0]) + (s[1] - s[0]) == bs for o, s in got[:-1])


def _numpy_scores(model, ent, rel, s, p, o):
    K = ent.shape[1]
    if model == "DistMult":
        return float(np.sum(ent[s] * rel[p] * ent[o]))
    h = K // 2
    sr, si, pr, pi, orr, oi = ent[s, :h], ent[s, h:], rel[p, :h], rel[p, h:], ent[o, :h], ent[o, h:]
    sc = float(np.sum(sr * (pr * orr + pi * oi) + si * (pr * oi - pi * orr)))
    return sc * 2.0 / (K / 2.0) if model == "HolE" else sc


def _numpy_loss(model, ent, rel, queries, labels, side, reduction, eps):
    n = ent.shape[0]
    total = 0.0
    for (s, p, o), lab in zip(queries, labels):
        row = 0.0
        for e in range(n):
            lg = _numpy_scores(model, ent, rel, e, p, o) if side == "s" else _numpy_scores(model, ent, rel, s, p, e)
            lg = min(max(lg, -75.0), 75.0)
            y = (1.0 - eps) * (e in lab) + eps / n
            row += np.log1p(np.exp(lg)) - y * lg
        total += row / n if reduction == "mean" else row
    return total


@pytest.mark.parametrize("model", ["DistMult", "ComplEx", "HolE"])
@pytest.mark.parametrize("side", ["o", "s"])
@pytest.mark.parametrize("reduction", ["sum", "mean"])
@pytest.mark.parametrize("eps", [0.0, 0.1])
def test_oracle_vs_numpy(model, side, reduction, eps):
    """Loss and central-difference gradients of the numpy restatement against the oracle, both float64; some logits
    are pushed past the clip so that their zero gradient is covered."""
    rng = np.random.default_rng(3)
    E, R, K = 5, 2, 4
    ent, rel = rng.uniform(-1, 1, (E, K)), rng.uniform(-1, 1, (R, K))
    queries = np.array([[0, 1, 3], [2, 0, 2], [4, 1, 0]])
    labels = [[3], [0, 2, 4], [0, 1, 2, 3, 4]]
    if model == "DistMult":
        ent[1] *= 40.0
        rel[1] *= 40.0
    for matmul in (False, True):
        loss, g_ent, g_rel = k_vs_all_oracle.loss_and_grads(model, ent, rel, queries, labels, side, reduction, eps,
                                                            matmul=matmul)
        assert loss == pytest.approx(_numpy_loss(model, ent, rel, queries, labels, side, reduction, eps), rel=1e-12)
        for table, grad in ((ent, g_ent), (rel, g_rel)):
            num = np.zeros_like(table)
            for idx in np.ndindex(*table.shape):
                h = 1e-6
                table[idx] += h
                up = _numpy_loss(model, ent, rel, queries, labels, side, reduction, eps)
                table[idx] -= 2 * h
                down = _numpy_loss(model, ent, rel, queries, labels, side, reduction, eps)
                table[idx] += h
                num[idx] = (up - down) / (2 * h)
            assert np.allclose(grad, num, rtol=1e-5, atol=1e-6), (matmul, np.abs(grad - num).max())


@pytest.mark.parametrize("model", ["DistMult", "ComplEx", "HolE"])
@pytest.mark.parametrize("side", ["o", "s"])
def test_oracle_is_the_reference_nll_on_two_entities(model, side):
    """eps = 0, n_ent = 2, one label per query: the loss is the reference's nll (eta = 1, reduction sum) of the label
    as the positive and the other entity as its corruption, summed over the batch."""
    rng = np.random.default_rng(5)
    K = 6
    ent, rel = rng.uniform(-2, 2, (2, K)), rng.uniform(-2, 2, (3, K))
    queries = np.array([[0, 0, 1], [1, 2, 1], [0, 1, 0], [1, 1, 0]])
    col = 2 if side == "o" else 0
    labels = [[int(q[col])] for q in queries]
    loss, _, _ = k_vs_all_oracle.loss_and_grads(model, ent, rel, queries, labels, side, "sum", 0.0)
    E, Rt = torch.as_tensor(ent), torch.as_tensor(rel)
    neg = queries.copy()
    neg[:, col] = 1 - neg[:, col]
    score = lambda t: ref_step.corruption_scores(model, "o", E[t[:, 0]], Rt[t[:, 1]], E[t[:, 0]], E)[
        torch.arange(len(t)), torch.as_tensor(t[:, 2])]
    sp, sn = score(queries), score(neg)
    want = float(ref_step.per_positive_loss("nll", sp, sn[None], reduction="sum").sum())
    assert loss == pytest.approx(want, rel=1e-12)
