"""CPU tests of NSCaching (DESIGN.md 3.20): the key rows and update flags of datasets.nscaching_tables against brute
force, the facade's refusals, the C struct's layout, and the restatement's selection law (Gumbel-top-1 draws a candidate
with probability softmax(score))."""
import ctypes as C
import math
import os
import subprocess
import tempfile

import numpy as np
import pytest

import nscaching_oracle as nsc
from ampligraph_b200 import _lib
from ampligraph_b200.datasets import FilterIndex, k_vs_all_queries, nscaching_tables


def _brute(t, batch_size):
    rows = {0: {}, 1: {}}
    key_rows = np.zeros((len(t), 2), np.int64)
    update = np.zeros((len(t), 2), np.uint8)
    for side, key in ((0, lambda x: (x[1], x[2])), (1, lambda x: (x[0], x[1]))):
        seen = set()
        for i, x in enumerate(t.tolist()):
            k = key(x)
            key_rows[i, side] = rows[side].setdefault(k, len(rows[side]))
            if (i // batch_size, k) not in seen:
                seen.add((i // batch_size, k))
                update[i, side] = 1
    return key_rows, update, (len(rows[0]), len(rows[1]))


@pytest.mark.parametrize("batch_size", [1, 7, 50, 64, 1000])
def test_key_rows_and_update_flags_against_brute_force(batch_size):
    """Keys repeat within and across batches (few entities and relations); 64 does not divide n = 300."""
    rng = np.random.default_rng(batch_size)
    E, R, n = 9, 3, 300
    t = np.stack([rng.integers(0, E, n), rng.integers(0, R, n), rng.integers(0, E, n)], 1).astype(np.int32)
    t[5] = t[3]  # the same triple twice in one batch
    got = nscaching_tables(t, E, R, batch_size)
    key_rows, update, n_keys = _brute(t, batch_size)
    assert got["key_rows"].dtype == np.int32 and got["update"].dtype == np.uint8
    assert (got["key_rows"] == key_rows).all() and (got["update"] == update).all()
    assert got["n_keys"] == n_keys and got["filter"] is None
    # the rows are KvsAll's query numbers
    for side, name in ((0, "s"), (1, "o")):
        q, _, _ = k_vs_all_queries(FilterIndex(t, E), t, name)
        assert len(q) == n_keys[side]
    if batch_size >= n:
        assert update.sum() == sum(n_keys)


def test_filter_arrays_are_the_filter_index():
    rng = np.random.default_rng(3)
    t = rng.integers(0, 6, (40, 3)).astype(np.int32)
    got = nscaching_tables(t, 6, 6, 10, filtered=True)
    f = FilterIndex(t, 6)
    for side, (keys, vals) in (("s", f._sub), ("o", f._obj)):
        assert (got["filter"][side][0] == keys).all() and (got["filter"][side][1] == vals).all()


def test_nscaching_struct_matches_header():
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "%s"\nint main(void){printf("%%zu %%zu %%zu %%zu %%zu\\n", '
           'sizeof(kge_nscaching), offsetof(kge_nscaching, sub_n_keys), offsetof(kge_nscaching, obj_n_keys), '
           'offsetof(kge_nscaching, obj_filter_n), offsetof(kge_nscaching, obj_filter_vals_dev)); return 0;}' % _lib.HEADER)
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "s.c"), "w").write(src)
        subprocess.check_call(["gcc", "-o", os.path.join(d, "s"), os.path.join(d, "s.c")])
        sizes = [int(x) for x in subprocess.check_output([os.path.join(d, "s")]).split()]
    S = _lib.KgeNSCaching
    assert [C.sizeof(S), S.sub_n_keys.offset, S.obj_n_keys.offset, S.obj_filter_n.offset,
            S.obj_filter_vals.offset] == sizes, sizes


def test_gumbel_top1_frequencies_are_softmax():
    """With N1 = 1 the refresh keeps argmax(score + G) over the valid candidates: over many (seed, step) pairs each of
    four fixed scores is kept with probability softmax(score).  2,000 draws: every frequency lies within 5 binomial
    standard deviations (<= 0.056) of its probability."""
    scores = np.array([0.0, 1.0, -1.0, 2.0])
    prob = np.exp(scores) / np.exp(scores).sum()
    n = 2000
    wins = np.zeros(4)
    for trial in range(n):
        seed, step = 1000 + trial, trial % 7
        keys = [scores[c] + nsc.gumbel(seed, step, 3, c, trial & 1) for c in range(4)]
        wins[int(np.argmax(keys))] += 1
    sigma = np.sqrt(prob * (1 - prob) / n)
    assert (np.abs(wins / n - prob) <= 5 * sigma).all(), (wins / n, prob)


def test_gumbel_uniform_is_exact_in_fp32_and_inside_the_open_interval():
    for w in (0, 1, 511, 512, 2 ** 31, MASK := 0xFFFFFFFF, MASK - 511):
        u = ((w >> 9) + 0.5) * 2.0 ** -23
        assert 0 < u < 1 and float(np.float32(u)) == u
        assert math.isfinite(-math.log(-math.log(u)))


def _model(**kw):
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    return ScoringBasedEmbeddingModel(eta=2, k=4, scoring_type=kw.pop("scoring_type", "TransE"), **kw)


X = np.array([["a", "r", "b"], ["b", "r", "c"], ["c", "q", "a"]])


@pytest.mark.parametrize("kw,match", [
    ({"negative_sampler": "uniform", "negative_sampler_params": {}}, "applies to negative_sampler='nscaching' only"),
    ({"negative_sampler": "bernoulli", "negative_sampler_params": {"cache_size": 5}}, "'nscaching' only"),
    ({"negative_sampler": "nscaching", "negative_sampler_params": [("cache_size", 5)]}, "must be a dict"),
    ({"negative_sampler": "nscaching", "negative_sampler_params": {"cache": 5}}, "unknown negative_sampler_params"),
    ({"negative_sampler": "nscaching", "negative_sampler_params": {"cache_size": 5.0}}, r"\['cache_size'\] must be an int"),
    ({"negative_sampler": "nscaching", "negative_sampler_params": {"random_size": True}}, "must be an int"),
    ({"negative_sampler": "nscaching", "negative_sampler_params": {"random_size": np.bool_(1)}}, "must be an int"),
    ({"negative_sampler": "nscaching", "negative_sampler_params": {"cache_size": 0}}, "cache_size >= 1"),
    ({"negative_sampler": "nscaching", "negative_sampler_params": {"random_size": -1}}, "random_size >= 1"),
    ({"negative_sampler": "nscaching", "negative_sampler_params": {"cache_size": 500, "random_size": 13}}, "<= 512"),
    ({"negative_sampler": "nscaching", "one_vs_all": "s,o"}, "sampled-training options"),
    ({"negative_sampler": "nscaching", "k_vs_all": "o"}, "sampled-training options"),
    ({"negative_sampler": "NSCaching"}, "negative_sampler must be one of"),
])
def test_fit_refusals(kw, match):
    """Refused with ValueError before anything is indexed (no data indexer is built) and without a GPU."""
    scoring = "DistMult" if ("one_vs_all" in kw or "k_vs_all" in kw) else "TransE"
    m = _model(scoring_type=scoring)
    m.compile(loss="multiclass_nll" if "one_vs_all" in kw else "nll")
    with pytest.raises(ValueError, match=match):
        m.fit(X, epochs=1, verbose=False, **kw)
    assert m.data_indexer is True and m.engine is None


def test_fit_accepts_int_params_of_numpy_type_before_indexing(monkeypatch):
    """np.int64 values pass the checks (the refusal comes from the next check, several GPUs)."""
    m = _model()
    m.compile(loss="pairwise")
    monkeypatch.setattr(type(m), "_world", lambda self: 2)
    with pytest.raises(NotImplementedError, match="single-GPU only"):
        m.fit(X, epochs=1, verbose=False, negative_sampler="nscaching",
              negative_sampler_params={"cache_size": np.int64(3), "random_size": 512 - 3})
    assert m.data_indexer is True and m.engine is None


def test_reciprocal_refusal_comes_first():
    m = _model(scoring_type="DistMult", reciprocal_relations=True)
    m.compile(loss="pairwise")
    with pytest.raises(NotImplementedError) as e:
        m.fit(X, epochs=1, verbose=False, negative_sampler="nscaching", negative_sampler_params={"cache": 1})
    assert str(e.value).startswith("reciprocal relations: fit trains against sampled corruptions")
