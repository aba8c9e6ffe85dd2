"""CPU tests of the negative sampler (DESIGN.md 3.18): its Python restatement against the corruption stream, the
per-fit tables of datasets.negative_sampler_tables, the C struct's layout, and the facade's refusals."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import negative_sampler_oracle as nso
from ampligraph_b200 import _lib
from ampligraph_b200.datasets import FilterIndex, negative_sampler_tables
from oracle import philox


def _triples(rng, E, R, n):
    return np.stack([rng.integers(0, E, n), rng.integers(0, R, n), rng.integers(0, E, n)], 1).astype(np.int32)


@pytest.mark.parametrize("B,eta,seed,step", [(1, 1, 0, 0), (37, 3, 5, 2), (50, 10, 2 ** 40 + 3, 2 ** 33 + 1)])
def test_uniform_oracle_is_the_corruption_stream(B, eta, seed, step):
    """No thresholds, pools or filter: attempt 0 is the draw of philox.corruption_stream, corruption for corruption."""
    rng = np.random.default_rng(B)
    E = 97
    t = _triples(rng, E, 5, B)
    repl, keep, misses = nso.sample(t, eta, E, seed, step)
    assert misses == 0
    assert (nso.corrupted_triples(t, eta, repl, keep) == philox.corruption_stream(t, eta, E, seed, step)).all()


def test_filtered_oracle_redraws_known_corruptions():
    """With max_attempts = 1 every known corruption is a miss and nothing changes; with more attempts only the entities
    of known corruptions change, the sides never, and what is still known is exactly the misses."""
    rng = np.random.default_rng(1)
    E, R, eta = 6, 2, 5
    train = _triples(rng, E, R, 30)
    t = train
    known = set(map(tuple, train.tolist()))
    r0, k0, m0 = nso.sample(t, eta, E, 3, 4)
    n_known = sum(tuple(x) in known for x in nso.corrupted_triples(t, eta, r0, k0).tolist())
    assert n_known > 10  # a dense graph: many collisions
    r1, k1, m1 = nso.sample(t, eta, E, 3, 4, train=train, max_attempts=1)
    assert (r1 == r0).all() and (k1 == k0).all() and m1 == n_known
    r5, k5, m5 = nso.sample(t, eta, E, 3, 4, train=train, max_attempts=5)
    assert (k5 == k0).all()
    still = [tuple(x) in known for x in nso.corrupted_triples(t, eta, r5, k5).tolist()]
    assert sum(still) == m5 < n_known
    changed = r5 != r0
    was_known = np.array([tuple(x) in known for x in nso.corrupted_triples(t, eta, r0, k0).tolist()])
    assert not (changed & ~was_known).any()


def test_bernoulli_thresholds_on_hand_built_relations():
    """t_p = floor(2^32 |T_p| / (|H_p| + |T_p|)) over distinct triples: 1-1, 1-N and N-1 relations, duplicates counted
    once, a relation without triples at 2^31."""
    t = np.array([
        [0, 0, 1], [2, 0, 3], [2, 0, 3],             # p0, 1-1: H = {0, 2}, T = {1, 3} (the duplicate counts once)
        [0, 1, 1], [0, 1, 2], [0, 1, 3], [0, 1, 3],  # p1, 1-N: H = {0}, T = {1, 2, 3}
        [1, 2, 0], [2, 2, 0], [3, 2, 0], [3, 2, 0],  # p2, N-1: H = {1, 2, 3}, T = {0}
        [4, 4, 5]], dtype=np.int32)                  # p3 has no triples; p4: H = {4}, T = {5}
    tab = negative_sampler_tables(t, 6, 5, "bernoulli")
    thr = tab["thresholds"]
    assert thr.dtype == np.uint32 and thr.shape == (5,)
    assert thr.tolist() == [2 ** 31, 3 * 2 ** 30, 2 ** 32 // 4, 2 ** 31, 2 ** 31]
    assert tab["pools"] is None and tab["filter"] is None
    # not a multiple of 1/2^32: floor, computed exactly
    t3 = np.array([[0, 0, 1], [0, 0, 2], [3, 0, 1]], dtype=np.int32)  # H = {0, 3}, T = {1, 2}
    t5 = np.array([[0, 0, 1], [0, 0, 2], [3, 0, 1], [4, 0, 1]], dtype=np.int32)  # H = {0, 3, 4}, T = {1, 2}
    assert negative_sampler_tables(t3, 5, 1, "bernoulli")["thresholds"].tolist() == [2 ** 31]
    assert negative_sampler_tables(t5, 5, 1, "bernoulli")["thresholds"].tolist() == [(2 << 32) // 5]


def test_pseudo_typed_pools():
    """The sorted distinct subjects (objects) of each relation as a CSR over all n_rel relations; empty rows where a
    relation has no triples."""
    rng = np.random.default_rng(2)
    E, R = 50, 6
    t = _triples(rng, E, R - 1, 300)  # relation R - 1 has no triples
    tab = negative_sampler_tables(np.concatenate([t, t[:20]]), E, R, "pseudo_typed")
    assert tab["thresholds"] is None and tab["filter"] is None
    for side, col in (("s", 0), ("o", 2)):
        off, ids = tab["pools"][side]
        assert off.dtype == np.int64 and ids.dtype == np.int32 and off.shape == (R + 1,) and off[0] == 0
        for p in range(R):
            want = np.unique(t[t[:, 1] == p, col])
            assert (ids[off[p]:off[p + 1]] == want).all(), (side, p)
        assert off[R] == off[R - 1] == len(ids)


def test_filter_arrays_are_the_filter_index():
    """The filter arrays are FilterIndex._sub (key p * n_ent + o, value s) and ._obj (key p * n_ent + s, value o) of
    the training triples: lexsorted, each known pair once."""
    rng = np.random.default_rng(3)
    E, R = 40, 4
    t = _triples(rng, E, R, 500)
    tab = negative_sampler_tables(t, E, R, "uniform", filtered=True)
    f = FilterIndex(t, E)
    for side, (want_k, want_v) in (("s", f._sub), ("o", f._obj)):
        keys, vals = tab["filter"][side]
        assert keys.dtype == np.int64 and vals.dtype == np.int32
        assert (keys == want_k).all() and (vals == want_v).all()
        pairs = keys * E + vals  # strictly increasing: lexsorted and distinct
        assert (np.diff(pairs) > 0).all()
    u = np.unique(t.astype(np.int64), axis=0)
    keys, vals = tab["filter"]["s"]
    assert (np.sort(keys * E + vals) == np.sort((u[:, 1] * E + u[:, 2]) * E + u[:, 0])).all()
    keys, vals = tab["filter"]["o"]
    assert (np.sort(keys * E + vals) == np.sort((u[:, 1] * E + u[:, 0]) * E + u[:, 2])).all()
    assert tab["thresholds"] is None and tab["pools"] is None
    assert negative_sampler_tables(t, E, R) == {"thresholds": None, "pools": None, "filter": None}
    with pytest.raises(ValueError):
        negative_sampler_tables(t, E, R, "typed")


def test_negative_sampler_struct_matches_header():
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "%s"\nint main(void){printf("%%zu %%zu %%zu\\n", '
           'sizeof(kge_negative_sampler), offsetof(kge_negative_sampler, obj_filter_n), '
           'offsetof(kge_negative_sampler, obj_filter_vals_dev)); return 0;}' % _lib.HEADER)
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "s.c"), "w").write(src)
        subprocess.check_call(["gcc", "-o", os.path.join(d, "s"), os.path.join(d, "s.c")])
        sizes = [int(x) for x in subprocess.check_output([os.path.join(d, "s")]).split()]
    S = _lib.KgeNegativeSampler
    assert [C.sizeof(S), S.obj_filter_n.offset, S.obj_filter_vals.offset] == sizes, sizes


def _model(**kw):
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    m = ScoringBasedEmbeddingModel(eta=2, k=4, scoring_type=kw.pop("scoring_type", "DistMult"), **kw)
    return m


X = np.array([["a", "r", "b"], ["b", "r", "c"], ["c", "q", "a"]])


@pytest.mark.parametrize("kw,exc,match", [
    ({"negative_sampler": "typed"}, ValueError, "negative_sampler must be one of"),
    ({"negative_sampler": None}, ValueError, "negative_sampler must be one of"),
    ({"filter_negatives": 1}, ValueError, "filter_negatives must be a bool"),
    ({"filter_negatives": np.bool_(True)}, ValueError, "filter_negatives must be a bool"),
    ({"negative_sampler": "bernoulli", "one_vs_all": "s,o"}, ValueError, "sampled-training options"),
    ({"filter_negatives": True, "one_vs_all": "o"}, ValueError, "sampled-training options"),
    ({"negative_sampler": "pseudo_typed", "k_vs_all": "o"}, ValueError, "sampled-training options"),
])
def test_fit_refusals(kw, exc, match):
    """Refused before anything is indexed (no data indexer is built) and without a GPU."""
    loss = "multiclass_nll" if "one_vs_all" in kw else "nll"
    m = _model()
    m.compile(loss=loss)
    with pytest.raises(exc, match=match):
        m.fit(X, epochs=1, verbose=False, **kw)
    assert m.data_indexer is True and m.engine is None


def test_fit_refuses_several_gpus(monkeypatch):
    m = _model()
    m.compile(loss="pairwise")
    monkeypatch.setattr(type(m), "_world", lambda self: 2)
    with pytest.raises(NotImplementedError, match="single-GPU only"):
        m.fit(X, epochs=1, verbose=False, negative_sampler="bernoulli")
    assert m.data_indexer is True and m.engine is None


@pytest.mark.parametrize("kw", [{}, {"negative_sampler": "bernoulli"}, {"filter_negatives": True},
                                {"negative_sampler": "nope"}])
def test_reciprocal_refusal_comes_first(kw):
    """A model with reciprocal relations refuses sampled training with its own message, whatever the sampler."""
    m = _model(reciprocal_relations=True)
    m.compile(loss="pairwise")
    with pytest.raises(NotImplementedError) as e:
        m.fit(X, epochs=1, verbose=False, **kw)
    assert str(e.value).startswith("reciprocal relations: fit trains against sampled corruptions")
