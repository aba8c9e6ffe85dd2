"""CPU tests of shared negatives (DESIGN.md 3.21): the restatement of the corruptions against the per-positive
samplers at C = 1, its chunk boundaries, the workspace formula, the C ABI's declarations, and the facade's refusals."""
import re
import subprocess

import numpy as np
import pytest

import negative_sampler_oracle as nso
import shared_negatives_oracle as sno
from ampligraph_b200 import _lib
from ampligraph_b200.engine import shared_negatives_workspace_bytes
from oracle import philox


def _triples(rng, E, R, n):
    return np.stack([rng.integers(0, E, n), rng.integers(0, R, n), rng.integers(0, E, n)], 1).astype(np.int32)


@pytest.mark.parametrize("B,eta,seed,step", [(1, 1, 0, 0), (37, 3, 5, 2), (50, 10, 2 ** 40 + 3, 2 ** 33 + 1)])
def test_chunk_one_is_the_uniform_stream(B, eta, seed, step):
    rng = np.random.default_rng(B)
    E = 97
    t = _triples(rng, E, 5, B)
    ne, nk = sno.sample(t, eta, E, seed, step, chunk=1)
    assert (nso.corrupted_triples(t, eta, ne, nk) == philox.corruption_stream(t, eta, E, seed, step)).all()
    repl, keep, _ = nso.sample(t, eta, E, seed, step)
    assert (ne == repl).all() and (nk == keep).all()


def test_chunk_one_is_the_bernoulli_sampler():
    rng = np.random.default_rng(4)
    E, R, B, eta = 61, 4, 29, 6
    t = _triples(rng, E, R, B)
    thr = np.array([0, 2 ** 31, 3 * 2 ** 30, 2 ** 32 - 1], np.uint32)
    ne, nk = sno.sample(t, eta, E, 9, 7, chunk=1, thresholds=thr)
    repl, keep, _ = nso.sample(t, eta, E, 9, 7, thresholds=thr)
    assert (ne == repl).all() and (nk == keep).all()
    assert (nk.reshape(eta, B)[:, t[:, 1] == 0] == 1).all()  # t_p = 0: never the subject


@pytest.mark.parametrize("B,C", [(10, 3), (10, 4), (7, 7), (5, 9), (12, 1), (33, 32)])
def test_chunk_boundaries(B, C):
    """Positives of one chunk share every candidate (the draw of the chunk's first positive); the sides stay the
    per-positive sampler's; the last chunk may be shorter and C > B is one chunk."""
    rng = np.random.default_rng(B * 100 + C)
    E, eta, seed, step = 1000, 5, 3, 11
    t = _triples(rng, E, 3, B)
    ne, nk = sno.sample(t, eta, E, seed, step, chunk=C)
    repl, keep, _ = nso.sample(t, eta, E, seed, step)
    ne, repl = ne.reshape(eta, B), repl.reshape(eta, B)
    assert (nk == keep).all()
    n_chunks = -(-B // C)
    assert sno.candidates(B, C, eta, E, seed, step).shape == (n_chunks, eta)
    for k in range(n_chunks):
        lo, hi = k * C, min((k + 1) * C, B)
        assert (ne[:, lo:hi] == repl[:, lo:lo + 1]).all()
    if C > 1 and B > C:  # distinct chunks draw distinct candidates (E = 1000, 5 draws each)
        assert (ne[:, 0] != ne[:, C]).any()


def test_workspace_formula():
    r16 = lambda n: (n + 15) // 16 * 16
    for B, eta in ((0, 1), (1, 1), (3, 7), (1024, 256), (27212, 256)):
        assert shared_negatives_workspace_bytes(B, eta) == r16(4 * B * eta) + r16(4 * B) + r16(B * eta)


def test_abi_declared_and_exported():
    header = open(_lib.HEADER).read()
    for name in ("kge_shared_negatives_workspace_bytes", "kge_shared_negatives_step"):
        assert re.search(r"\b%s\(" % name, header), name
        assert name in _lib.PROTOTYPES
    so = _lib.SO_PATH
    syms = subprocess.check_output(["nm", "-D", "--defined-only", so], text=True)
    for name in ("kge_shared_negatives_workspace_bytes", "kge_shared_negatives_step"):
        assert re.search(r"\bT %s$" % name, syms, re.M), name


def _model(**kw):
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    return ScoringBasedEmbeddingModel(eta=2, k=4, scoring_type=kw.pop("scoring_type", "TransE"), **kw)


X = np.array([["a", "r", "b"], ["b", "r", "c"], ["c", "q", "a"]])


@pytest.mark.parametrize("kw,exc,match", [
    ({"shared_negatives": True}, ValueError, "shared_negatives must be an int >= 0"),
    ({"shared_negatives": np.bool_(True)}, ValueError, "shared_negatives must be an int >= 0"),
    ({"shared_negatives": 2.0}, ValueError, "shared_negatives must be an int >= 0"),
    ({"shared_negatives": "4"}, ValueError, "shared_negatives must be an int >= 0"),
    ({"shared_negatives": -1}, ValueError, "shared_negatives must be an int >= 0"),
    ({"shared_negatives": 4, "one_vs_all": "s,o"}, ValueError, "cannot be combined with one_vs_all or k_vs_all"),
    ({"shared_negatives": 4, "k_vs_all": "o"}, ValueError, "cannot be combined with one_vs_all or k_vs_all"),
    ({"shared_negatives": 4, "negative_sampler": "pseudo_typed"}, ValueError, "picks entities per positive"),
    ({"shared_negatives": 4, "negative_sampler": "nscaching"}, ValueError, "picks entities per positive"),
    ({"shared_negatives": 4, "filter_negatives": True}, ValueError, "picks entities per positive"),
    ({"shared_negatives": 4, "focusE": True}, NotImplementedError, "user losses and focusE"),
])
def test_fit_refusals(kw, exc, match):
    """Refused before anything is indexed (no data indexer is built) and without a GPU."""
    scoring = "DistMult" if ("one_vs_all" in kw or "k_vs_all" in kw) else "TransE"
    m = _model(scoring_type=scoring)
    m.compile(loss="multiclass_nll" if "one_vs_all" in kw else "nll")
    with pytest.raises(exc, match=match):
        m.fit(X, epochs=1, verbose=False, **kw)
    assert m.data_indexer is True and m.engine is None


def test_fit_refuses_user_loss():
    m = _model()
    m.compile(loss=lambda sp, sn: (sn - sp).clamp(min=0).sum())
    with pytest.raises(NotImplementedError, match="user losses and focusE"):
        m.fit(X, epochs=1, verbose=False, shared_negatives=2)
    assert m.data_indexer is True and m.engine is None


def test_fit_refuses_several_gpus(monkeypatch):
    m = _model()
    m.compile(loss="pairwise")
    monkeypatch.setattr(type(m), "_world", lambda self: 2)
    with pytest.raises(NotImplementedError, match="single-GPU only"):
        m.fit(X, epochs=1, verbose=False, shared_negatives=np.int64(2))
    assert m.data_indexer is True and m.engine is None


def test_reciprocal_refusal_comes_first():
    m = _model(scoring_type="DistMult", reciprocal_relations=True)
    m.compile(loss="pairwise")
    with pytest.raises(NotImplementedError) as e:
        m.fit(X, epochs=1, verbose=False, shared_negatives=True)
    assert str(e.value).startswith("reciprocal relations: fit trains against sampled corruptions")
