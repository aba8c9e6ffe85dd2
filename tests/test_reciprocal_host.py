"""CPU tests of reciprocal relations (DESIGN.md 3.17): every refusal, the remap helper datasets.reciprocal_triples
against a numpy loop (inverse triples, the per-batch layout of 1vsAll rows, KvsAll side-s queries as side-o queries
with the same labels), the relation initializer's shape, the saved flag, and select_best_model_ranking's grid key."""
import pickle

import numpy as np
import pytest
import torch

from ampligraph_b200.datasets import FilterIndex, k_vs_all_queries, reciprocal_triples

X = np.array([["a", "r", "b"], ["b", "r", "c"], ["c", "q", "a"], ["a", "q", "c"]])


def _model(scoring="ComplEx", loss="multiclass_nll", reg=None, init="glorot_uniform", reciprocal=True, **kw):
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    m = ScoringBasedEmbeddingModel(eta=2, k=4, scoring_type=scoring, reciprocal_relations=reciprocal, **kw)
    m.compile(optimizer="adam", loss=loss, entity_relation_regularizer=reg, entity_relation_initializer=init)
    return m


def _untouched(m):
    assert m.engine is None and m.data_indexer is True  # nothing was indexed or built


# ---------------------------------------------------------------- refusals
@pytest.mark.parametrize("scoring", ["TransE", "RotatE"])
def test_distance_models_refused(scoring):
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    with pytest.raises(NotImplementedError, match="reciprocal relations.*%s" % scoring):
        ScoringBasedEmbeddingModel(eta=2, k=4, scoring_type=scoring, reciprocal_relations=True)
    ScoringBasedEmbeddingModel(eta=2, k=4, scoring_type=scoring)  # the default is unchanged


@pytest.mark.parametrize("scoring", ["DistMult", "ComplEx", "HolE"])
def test_trilinear_models_accepted(scoring):
    assert _model(scoring).reciprocal_relations
    assert not _model(scoring, reciprocal=False).reciprocal_relations


def test_sampled_training_refused():
    m = _model(loss="pairwise")
    for call in (lambda: m.fit(X, epochs=1), lambda: m.train_on_batch(X),
                 lambda: m.train_on_batches([np.zeros((2, 3), np.int32)])):
        with pytest.raises(NotImplementedError, match="reciprocal relations.*sampled corruptions"):
            call()
    _untouched(m)


def test_focuse_refused():
    m = _model()
    Xw = np.concatenate([X, np.ones((len(X), 1), dtype=X.dtype)], 1)
    for kw in ({"one_vs_all": "s,o"}, {}):
        with pytest.raises(NotImplementedError, match="reciprocal relations"):
            m.fit(Xw, epochs=1, focusE=True, **kw)
    _untouched(m)


def test_user_loss_refused():
    from ampligraph_b200.latent_features import loss_functions
    m = _model()
    m.compile(optimizer="adam", loss=loss_functions.LossFunctionWrapper(lambda p, n: (n - p).sum(), "user"))
    with pytest.raises(NotImplementedError, match="reciprocal relations: a user loss"):
        m.fit(X, epochs=1, one_vs_all="s,o")
    _untouched(m)


def test_relation_prediction_refused():
    m = _model()
    with pytest.raises(NotImplementedError, match="reciprocal relations: the relation-prediction term"):
        m.fit(X, epochs=1, one_vs_all="s,o", relation_prediction_weight=0.5)
    _untouched(m)


def test_several_gpus_refused(monkeypatch):
    from ampligraph_b200.latent_features import models
    monkeypatch.setattr(models.ScoringBasedEmbeddingModel, "_world", lambda self: 2)
    m = _model()
    m.distributed = True
    for kw in ({"one_vs_all": "s,o"}, {"k_vs_all": "o"}):
        if "k_vs_all" in kw:
            m.compile(optimizer="adam", loss="nll")
        with pytest.raises(NotImplementedError, match="reciprocal relations: training is single-GPU only"):
            m.fit(X, epochs=1, **kw)
    _untouched(m)
    m.is_fitted = True
    with pytest.raises(NotImplementedError, match="reciprocal relations: evaluate is single-GPU only"):
        m.evaluate(X)


def test_relation_ids_of_inverse_rows_refused():
    m = _model(max_rel_size=3, max_ent_size=5)
    m.data_indexer = False
    ids = np.array([[0, 2, 1], [1, 3, 2]])
    with pytest.raises(ValueError, match="relation ids must be below max_rel_size = 3"):
        m._index(ids)
    assert m._index(ids[:1]).tolist() == [[0, 2, 1]]
    plain = _model(max_rel_size=3, max_ent_size=5, reciprocal=False)
    plain.data_indexer = False
    assert plain._index(ids).tolist() == ids.tolist()  # without reciprocal relations nothing changes


def test_r_inv_refused_on_a_plain_model():
    m = _model(reciprocal=False)
    m.is_fitted = True
    with pytest.raises(ValueError, match="r_inv.*reciprocal relations"):
        m.get_embeddings(["r"], "r_inv")


# ---------------------------------------------------------------- remap helper
def _inverse_loop(t, R):
    return np.array([[o, p + R, s] for s, p, o in np.asarray(t).tolist()], np.int32).reshape(-1, 3)


@pytest.mark.parametrize("n,bs", [(0, 4), (1, 4), (7, 3), (12, 4), (10, 1000), (9, 1)])
@pytest.mark.parametrize("sides", ["s,o", "o", "s"])
def test_rows_against_a_loop(n, bs, sides):
    rng = np.random.default_rng(n * 31 + bs)
    R = 5
    t = np.stack([rng.integers(0, 9, n), rng.integers(0, R, n), rng.integers(0, 9, n)], 1).astype(np.int32)
    want = []
    for lo in range(0, n, bs):
        b = t[lo:lo + bs]
        want += ([b] if "o" in sides else []) + ([_inverse_loop(b, R)] if "s" in sides else [])
    want = np.concatenate(want) if want else np.zeros((0, 3), np.int32)
    got = reciprocal_triples(t, R, sides, bs)
    assert got.dtype == np.int32 and got.flags.c_contiguous and np.array_equal(got, want)
    m = len(sides.split(","))
    for lo in range(0, n, bs):  # fit's slice of batch lo // bs
        b = t[lo:lo + bs]
        want_b = np.concatenate(([b] if "o" in sides else []) + ([_inverse_loop(b, R)] if "s" in sides else []))
        assert np.array_equal(got[m * lo:m * (lo + bs)], want_b)
    assert np.array_equal(reciprocal_triples(t, R, "s"), _inverse_loop(t, R))
    assert np.array_equal(reciprocal_triples(t, R, "s,o"), np.concatenate([t, _inverse_loop(t, R)]).reshape(-1, 3))


def test_k_vs_all_side_s_queries_become_side_o_queries():
    """Each side-s query (p, o) with labels {s} is the side-o query (o, p + R) of the inverse triples, with the same
    label list: the labels an object query of the inverse triples would have."""
    rng = np.random.default_rng(3)
    E, R, n = 11, 4, 60
    t = np.stack([rng.integers(0, E, n), rng.integers(0, R, n), rng.integers(0, E, n)], 1)
    q_s, off_s, ids_s = k_vs_all_queries(FilterIndex(t, E), t, "s")
    q = reciprocal_triples(q_s, R, "s")
    inv = _inverse_loop(t, R)
    labels = {}
    for s, p, o in inv.tolist():
        labels.setdefault((s, p), set()).add(o)
    assert len(q) == len(labels)
    for i, (s, p, o) in enumerate(q.tolist()):
        assert R <= p < 2 * R and o == ids_s[off_s[i]]
        assert ids_s[off_s[i]:off_s[i + 1]].tolist() == sorted(labels[(s, p)])
    q_o, off_o, ids_o = k_vs_all_queries(FilterIndex(inv, E), inv, "o")  # the same queries, in the same order
    assert np.array_equal(q_o, q) and np.array_equal(off_o, off_s) and np.array_equal(ids_o, ids_s)


def test_filter_lists_of_the_inverse():
    """evaluate and top-n keep the side-s filter: lookup(t, 's') lists, for (s, p, o), what lookup(inverse, 'o') lists
    over the inverse triples."""
    rng = np.random.default_rng(4)
    E, R, n = 9, 3, 40
    t = np.stack([rng.integers(0, E, n), rng.integers(0, R, n), rng.integers(0, E, n)], 1)
    inv = _inverse_loop(t, R)
    a = FilterIndex(t, E).lookup(t, "s")
    b = FilterIndex(inv, E).lookup(inv, "o")
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


# ---------------------------------------------------------------- initializers
class _FakeEngine:
    seen = {}

    def __init__(self, scoring_type, k, eta, n_ent, n_rel, **kw):
        _FakeEngine.seen = {"n_ent": n_ent, "n_rel": n_rel}
        self.n_ent, self.n_rel = n_ent, n_rel

    def set_embeddings(self, ent, rel):
        _FakeEngine.seen.update(ent=ent, rel=rel)

    def __getattr__(self, name):
        return lambda *a, **k: None


def test_engine_and_initializers_see_2r_rows(monkeypatch):
    from ampligraph_b200.latent_features import models
    monkeypatch.setattr(models, "KGEEngine", _FakeEngine)
    shapes = []

    def init(shape):
        shapes.append(shape)
        return np.zeros(shape, np.float32)
    m = _model("DistMult", init=init)
    m.max_ent_size, m.max_rel_size = 6, 3
    m._build_engine()
    assert _FakeEngine.seen["n_rel"] == 6 and shapes == [(6, 4), (6, 4)]
    m = _model("ComplEx", init=[np.zeros((6, 8)), np.ones((6, 8))])
    m.max_ent_size, m.max_rel_size = 6, 3
    m._build_engine()
    assert _FakeEngine.seen["rel"].shape == (6, 8)
    plain = _model("ComplEx", reciprocal=False, init=init)
    plain.max_ent_size, plain.max_rel_size = 6, 3
    plain._build_engine()
    assert _FakeEngine.seen["n_rel"] == 3


def test_ndarray_initializer_of_r_rows_refused(monkeypatch):
    from ampligraph_b200.latent_features import models
    monkeypatch.setattr(models, "KGEEngine", _FakeEngine)
    m = _model("ComplEx", init=[np.zeros((6, 8)), np.ones((3, 8))])
    m.max_ent_size, m.max_rel_size = 6, 3
    with pytest.raises(ValueError, match=r"needs shape \(6, 8\).*got shape \(3, 8\)"):
        m._build_engine()


# ---------------------------------------------------------------- save / load
class _SavedEngine:
    def __init__(self, R):
        self.t, self.slots = 3, {}
        self.tables = (torch.zeros((4, 8)), torch.arange(2 * R * 8, dtype=torch.float32).reshape(2 * R, 8))

    def get_embeddings(self):
        return self.tables


def test_flag_round_trip(monkeypatch, tmp_path):
    from ampligraph_b200.latent_features import models
    monkeypatch.setattr(models, "KGEEngine", _FakeEngine)
    m = _model()
    m.max_ent_size, m.max_rel_size, m.engine = 4, 2, _SavedEngine(2)
    path = str(tmp_path / "w.pkl")
    m.save_weights(path)
    with open(path, "rb") as f:
        assert pickle.load(f)["reciprocal_relations"] is True
    back = _model()
    back.load_weights(path)
    assert back.is_fitted and _FakeEngine.seen["n_rel"] == 4 and _FakeEngine.seen["rel"].shape == (4, 8)
    with pytest.raises(ValueError, match="reciprocal_relations=True, this model has False"):
        _model(reciprocal=False).load_weights(path)


def test_old_pickle_loads_as_plain(monkeypatch, tmp_path):
    """Files written before the flag existed have no such key: they load into plain models only."""
    from ampligraph_b200.latent_features import models
    monkeypatch.setattr(models, "KGEEngine", _FakeEngine)
    state = {"ent": np.zeros((4, 8), np.float32), "rel": np.zeros((2, 8), np.float32), "t": 1, "step": 1, "slots": {},
             "indexer": True, "max_ent_size": 4, "max_rel_size": 2}
    path = str(tmp_path / "old.pkl")
    with open(path, "wb") as f:
        pickle.dump(state, f)
    plain = _model(reciprocal=False)
    plain.load_weights(path)
    assert plain.is_fitted and _FakeEngine.seen["n_rel"] == 2
    with pytest.raises(ValueError, match="reciprocal_relations=False, this model has True"):
        _model().load_weights(path)


# ---------------------------------------------------------------- grid
def test_grid_key():
    from ampligraph_b200.evaluation import _build_model
    assert _build_model("ComplEx", {"k": 8, "reciprocal_relations": True}, 2).reciprocal_relations
    assert not _build_model("ComplEx", {"k": 8}, 2).reciprocal_relations
