"""Reciprocal relations on the GPU (DESIGN.md 3.17).  The oracle is the plain engine with 2R relation rows run on
explicitly remapped triples: a reciprocal step is one side-o 1vsAll or KvsAll call over the forward and inverse rows,
and a reciprocal subject rank is an object rank of the inverse triple.

- Steps (1vsAll, KvsAll, with N3 / DURA): the gradient tables and the loss that fit's step hands to the optimizer equal
  the plain engine's on the remapped rows: bit for bit on gated tables where every fp32 operation is exact, so the
  order of the REDs does not matter; to fp32 rounding where it is not (HolE's scale, the regularisers' large terms);
  and within the float64 oracle's per-element bound on random tables.
- fit end to end against a hand-written loop of plain-engine steps, and validation inside fit.
- evaluate, query_topn / query_topn_batch against a plain model sharing the tables, and discover_facts."""
import numpy as np
import pytest
import torch

import exact_oracle as xo
import k_vs_all_oracle
import one_vs_all_oracle
from ampligraph_b200 import discovery
from ampligraph_b200.datasets import FilterIndex, k_vs_all_queries, reciprocal_triples
from ampligraph_b200.engine import KGEEngine
from ampligraph_b200.latent_features import EarlyStopping, ScoringBasedEmbeddingModel
from test_gpu_one_vs_all_exact import _grads, exact_value, gated_tables

pytestmark = pytest.mark.gpu

MODELS = ["DistMult", "ComplEx", "HolE"]


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a)).cuda().contiguous()


def _model(scoring, k, E, R, ent, rel, loss="multiclass_nll", optimizer="sgd", reg=None, reciprocal=True, seed=0):
    """A model on integer ids (use_indexer=False) whose tables start as ent / rel."""
    m = ScoringBasedEmbeddingModel(eta=1, k=k, scoring_type=scoring, seed=seed, max_ent_size=E, max_rel_size=R,
                                   reciprocal_relations=reciprocal)
    m.data_indexer = False
    m.compile(optimizer=optimizer, loss=loss, entity_relation_initializer=[ent, rel], entity_relation_regularizer=reg)
    return m


def _plain_engine(scoring, k, E, ent, rel, loss="multiclass_nll", optimizer="sgd", reg=None, reduction="sum"):
    """The plain engine of _model's tables: rel has 2R rows, row p + R the inverse of p."""
    from ampligraph_b200.latent_features import optimizers, regularizers
    opt = optimizers.get(optimizer)
    eng = KGEEngine(scoring, k, 1, E, rel.shape[0], loss=loss, loss_params={"reduction": reduction},
                    optimizer=opt.name, optimizer_params=opt.hyperparams,
                    regularizer=[r.kernel_params() if r is not None else None for r in regularizers.get_pair(reg)])
    eng.set_embeddings(ent, rel)
    return eng


class _Steps:
    """Records, at every apply_gradients, the gradient tables and both loss slots the step hands to the optimizer."""

    def __init__(self, monkeypatch):
        self.seen = []
        apply = KGEEngine.apply_gradients

        def spy(eng):
            torch.cuda.synchronize()
            self.seen.append((*_grads(eng), eng.loss_acc.cpu().numpy().copy()))
            apply(eng)
        monkeypatch.setattr(KGEEngine, "apply_gradients", spy)


def _model_step(monkeypatch, m, x, **fit_kw):
    """One fit step of model m over all of x -> (g_ent, g_rel, loss slots)."""
    steps = _Steps(monkeypatch)
    m.fit(x, batch_size=1 << 20, epochs=1, verbose=False, **fit_kw)
    assert len(steps.seen) == 1
    monkeypatch.undo()
    return steps.seen[0]


def _plain_step(eng, calls):
    for call in calls:
        call(eng)
    torch.cuda.synchronize()
    out = (*_grads(eng), eng.loss_acc.cpu().numpy().copy())
    eng.close()
    return out


def _ova_rows(t, R, sides):
    """fit(one_vs_all=sides)'s rows of one batch, written out: forward rows, then inverse rows."""
    parts = ([t] if "o" in sides.split(",") else []) + ([np.stack([t[:, 2], t[:, 1] + R, t[:, 0]], 1)]
                                                        if "s" in sides.split(",") else [])
    return np.concatenate(parts).astype(np.int32)


# ---------------------------------------------------------------- 1vsAll step
def _gated_case(model, k, rng, G=5, g=16, B=60, R=3):
    """Gated tables (test_gpu_one_vs_all_exact) with 2R relation rows; targets outside the kept entity's group on both
    sides, so every row of either direction has (G - 1) g live candidates, a power of two."""
    group = np.repeat(np.arange(G), g)
    E = G * g
    s = rng.integers(0, E, B)
    o = (s + g * rng.integers(1, G, B)) % E
    t = np.stack([s, rng.integers(0, R, B), o], 1).astype(np.int32)
    ent, rel = gated_tables(model, k, G, group, 2 * R, rng)
    return E, R, ent, rel, t


@pytest.mark.parametrize("sides", ["s,o", "o", "s"])
@pytest.mark.parametrize("model", ["DistMult", "ComplEx"])
def test_one_vs_all_step_bit_exact(monkeypatch, model, sides):
    k = 36
    E, R, ent, rel, t = _gated_case(model, k, np.random.default_rng(len(sides) + len(model)))
    got = _model_step(monkeypatch, _model(model, k, E, R, ent, rel), t, one_vs_all=sides)
    rows = _ova_rows(t, R, sides)
    want = _plain_step(_plain_engine(model, k, E, ent, rel), [lambda e: e.one_vs_all_backward(_dev(rows), "o")])
    for a, b in zip(got, want):
        assert np.array_equal(a, b)
    _, want_ent, want_rel = one_vs_all_oracle.loss_and_grads(model, ent, rel, rows, "o", "sum", matmul=True)
    assert np.array_equal(got[0], exact_value(want_ent)) and np.array_equal(got[1], exact_value(want_rel))


@pytest.mark.parametrize("reduction", ["sum", "mean"])
@pytest.mark.parametrize("sides", ["s,o", "o", "s"])
@pytest.mark.parametrize("model", MODELS)
def test_one_vs_all_step_bound(monkeypatch, model, sides, reduction):
    rng = np.random.default_rng(len(model) * 7 + len(sides) + len(reduction))
    k, E, R, B = 24, 300, 5, 90
    K = xo.internal_k(model, k)
    ent = rng.uniform(-0.4, 0.4, (E, K)).astype(np.float32)
    rel = rng.uniform(-0.4, 0.4, (2 * R, K)).astype(np.float32)
    t = np.stack([rng.integers(0, E, B), rng.integers(0, R, B), rng.integers(0, E, B)], 1).astype(np.int32)
    from ampligraph_b200.latent_features import loss_functions
    loss = loss_functions.get("multiclass_nll", {"reduction": reduction})
    g_ent, g_rel, slots = _model_step(monkeypatch, _model(model, k, E, R, ent, rel, loss=loss), t, one_vs_all=sides)
    rows = _ova_rows(t, R, sides)
    want_loss, want_ent, want_rel = one_vs_all_oracle.loss_and_grads(model, ent, rel, rows, "o", reduction, matmul=True)
    bound = xo.OvaBound(model, ent, rel, rows)
    bound.add_side(rows, "o", reduction)
    where = (model, sides, reduction)
    bound.check_loss(float(slots[0]), want_loss, where)
    bound.check(g_ent, g_rel, want_ent, want_rel, where)
    assert not g_rel[R:].any() if sides == "o" else g_rel[R:].any()  # the inverse rows train exactly when 's' does
    assert not g_rel[:R].any() if sides == "s" else g_rel[:R].any()


# ---------------------------------------------------------------- KvsAll step
# (model, k, G, g, reduction, eps): n_ent = G g, a power of two under mean or eps > 0 (test_bit_exact_k_vs_all)
KVA = [("DistMult", 36, 5, 16, "sum", 0.0), ("ComplEx", 36, 4, 16, "mean", 0.5), ("DistMult", 36, 8, 16, "sum", 0.5),
       ("HolE", 36, 4, 16, "mean", 0.0)]


@pytest.mark.parametrize("sides", ["s,o", "o", "s"])
@pytest.mark.parametrize("case", KVA, ids=["-".join(map(str, c)) for c in KVA])
def test_k_vs_all_step(monkeypatch, case, sides):
    """Against the plain engine's explicit calls (side o's queries, then the inverse side-s queries as side-o
    queries) and the float64 oracle.  On the gated tables of DistMult and ComplEx every operation is exact: bit for bit
    with both.  HolE's logit scale 4 / K is not dyadic, so its REDs may round in either order: within fp32 rounding
    of the plain engine and within the oracle's bound."""
    model, k, G, g, reduction, eps = case
    rng = np.random.default_rng(G * g + len(sides))
    E, R, B = G * g, 3, 120
    ent, rel = gated_tables(model, k, G, np.repeat(np.arange(G), g), 2 * R, rng)
    t = np.stack([rng.integers(0, E, B), rng.integers(0, R, B), rng.integers(0, E, B)], 1).astype(np.int32)
    from ampligraph_b200.latent_features import loss_functions
    loss = loss_functions.get("nll", {"reduction": reduction})
    got = _model_step(monkeypatch, _model(model, k, E, R, ent, rel, loss=loss), t, k_vs_all=sides, label_smoothing=eps)
    findex = FilterIndex(t, E)
    queries = []
    for side in sides.split(","):
        q, off, ids = k_vs_all_queries(findex, t, side)
        if side == "s":
            q = np.stack([q[:, 2], q[:, 1] + R, q[:, 0]], 1).astype(np.int32)
        queries.append((q, off, ids))
    calls = [lambda e, q=q, off=off, ids=ids: e.k_vs_all_backward(_dev(q), "o", _dev(off), _dev(ids), eps)
             for q, off, ids in queries]
    want = _plain_step(_plain_engine(model, k, E, ent, rel, loss="nll", reduction=reduction), calls)
    for a, b in zip(got, want):
        if model == "HolE":
            np.testing.assert_allclose(a, b, rtol=1e-6, atol=1e-6 * np.abs(b).max())
        else:
            assert np.array_equal(a, b)
    want_ent = np.zeros_like(ent, np.float64)
    want_rel = np.zeros_like(rel, np.float64)
    bound = xo.OvaBound(model, ent, rel, np.concatenate([q for q, _, _ in queries]))
    for q, off, ids in queries:
        labels = [ids[off[i]:off[i + 1]] for i in range(len(q))]
        _, ge, gr = k_vs_all_oracle.loss_and_grads(model, ent, rel, q, labels, "o", reduction, eps, matmul=True)
        want_ent += ge
        want_rel += gr
        bound.add_side(q, "o", reduction, labels=labels, eps=eps)
    if model == "HolE":
        bound.check(got[0], got[1], want_ent, want_rel, case)
    else:
        assert np.array_equal(got[0], exact_value(want_ent)) and np.array_equal(got[1], exact_value(want_rel))


# ---------------------------------------------------------------- N3 and DURA
@pytest.mark.parametrize("reg", ["N3", "DURA"])
@pytest.mark.parametrize("model", ["DistMult", "ComplEx"])
def test_per_occurrence_regularisers_take_the_trained_rows(monkeypatch, model, reg):
    """With 1vsAll 's,o' the regulariser's term (loss slot 1) and gradients are n3_backward / dura_backward's on the
    2B remapped rows.  The regulariser's large terms on the gated tables' -128 gates make its REDs round, so the
    gradient tables agree to fp32 rounding and the fp64 loss slots to fp64 rounding."""
    from ampligraph_b200.latent_features import regularizers
    k = 36
    E, R, ent, rel, t = _gated_case(model, k, np.random.default_rng(11 + len(reg)))
    r = regularizers.get(reg, {"lambda": 0.25})
    got = _model_step(monkeypatch, _model(model, k, E, R, ent, rel, reg=r), t, one_vs_all="s,o")
    rows = _dev(_ova_rows(t, R, "s,o"))
    per_row_of = (lambda e, x: e.n3_backward(x)) if reg == "N3" else (lambda e, x: e.dura_backward(x))
    per_row = lambda e: per_row_of(e, rows)  # noqa: E731
    want = _plain_step(_plain_engine(model, k, E, ent, rel, reg=r),
                       [lambda e: e.one_vs_all_backward(rows, "o"), per_row])
    for a, b in zip(got[:2], want[:2]):
        np.testing.assert_allclose(a, b, rtol=1e-6, atol=1e-6 * np.abs(b).max())
    np.testing.assert_allclose(got[2], want[2], rtol=1e-12)
    alone = _plain_step(_plain_engine(model, k, E, ent, rel, reg=r), [per_row])
    half = _plain_step(_plain_engine(model, k, E, ent, rel, reg=r), [lambda e: per_row_of(e, rows[:len(t)])])
    assert got[2][1] == pytest.approx(alone[2][1], rel=1e-12) and got[2][1] > half[2][1] > 0


# ---------------------------------------------------------------- fit end to end
def test_fit_against_a_loop_of_plain_steps():
    """Three epochs of reciprocal ComplEx + N3 with 1vsAll 's,o' and Adam, four batches each (the last one short),
    against the same steps written out on a plain engine with 2R relations.  Both sum the same values with
    order-dependent REDs, so the tables and losses agree to fp32 rounding, not bit for bit."""
    from ampligraph_b200.latent_features import regularizers
    rng = np.random.default_rng(5)
    k, E, R, n, bs, epochs = 20, 150, 4, 350, 100, 3
    K = 2 * k
    ent = rng.uniform(-0.3, 0.3, (E, K)).astype(np.float32)
    rel = rng.uniform(-0.3, 0.3, (2 * R, K)).astype(np.float32)
    t = np.stack([rng.integers(0, E, n), rng.integers(0, R, n), rng.integers(0, E, n)], 1).astype(np.int32)
    reg = regularizers.get("N3", {"lambda": 0.01})
    m = _model("ComplEx", k, E, R, ent, rel, optimizer="adam", reg=reg)
    history = m.fit(t, batch_size=bs, epochs=epochs, verbose=False, one_vs_all="s,o").history["loss"]
    eng = _plain_engine("ComplEx", k, E, ent, rel, optimizer="adam", reg=reg)
    want, total, steps = [], 0.0, 0
    for _ in range(epochs):
        for lo in range(0, n, bs):
            rows = _dev(reciprocal_triples(t[lo:lo + bs], R, "s,o"))
            eng.one_vs_all_backward(rows, "o", step=steps)
            eng.n3_backward(rows, step=steps)
            eng.apply_gradients()
            steps += 1
        total += eng.read_loss()
        want.append(total / steps)
    np.testing.assert_allclose(history, want, rtol=1e-5)
    got_ent, got_rel = (a.cpu().numpy() for a in m.engine.get_embeddings())
    want_ent, want_rel = (a.cpu().numpy() for a in eng.get_embeddings())
    np.testing.assert_allclose(got_ent, want_ent, rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(got_rel, want_rel, rtol=1e-4, atol=1e-5)
    eng.close()


def _trained(scoring="ComplEx", k=16, E=120, R=5, n=600, seed=2):
    """A briefly trained reciprocal model on integer ids, its training triples and a plain model sharing its tables
    (2R relation rows)."""
    rng = np.random.default_rng(seed)
    t = np.stack([rng.integers(0, E, n), rng.integers(0, R, n), rng.integers(0, E, n)], 1).astype(np.int32)
    K = xo.internal_k(scoring, k)
    m = _model(scoring, k, E, R, rng.uniform(-0.3, 0.3, (E, K)).astype(np.float32),
               rng.uniform(-0.3, 0.3, (2 * R, K)).astype(np.float32), optimizer="adam")
    m.fit(t, batch_size=200, epochs=3, verbose=False, one_vs_all="s,o")
    ent, rel = (a.cpu().numpy() for a in m.engine.get_embeddings())
    plain = _model(scoring, k, E, 2 * R, ent, rel, reciprocal=False)
    plain._build_engine()
    plain.is_fitted = True
    return m, plain, t, ent, rel


def _inv(t, R):
    return reciprocal_triples(t, R, "s")


# ---------------------------------------------------------------- evaluate
@pytest.mark.parametrize("strategy", ["worst", "best", "middle"])
def test_evaluate_subject_side_is_the_inverse_object_side(strategy):
    m, plain, t, ent, rel = _trained()
    R = m.max_rel_size
    test = t[::7]
    subset = np.arange(0, m.max_ent_size, 3)
    subset = np.union1d(subset, test[:, [0, 2]].ravel())
    for use_filter in (False, {"train": t}):
        pf = {"train": _inv(t, R)} if use_filter else False
        for sub in (None, subset):
            kw = dict(use_filter=use_filter, entities_subset=sub, ranking_strategy=strategy, verbose=False)
            pkw = dict(kw, use_filter=pf)
            s = plain.evaluate(_inv(test, R), corrupt_side="o", **pkw)
            o = plain.evaluate(test, corrupt_side="o", **kw)  # side o keeps the forward rows and filter
            assert np.array_equal(m.evaluate(test, corrupt_side="s", **kw), s)
            assert np.array_equal(m.evaluate(test, corrupt_side="o", **kw), o)
            assert np.array_equal(m.evaluate(test, corrupt_side="s,o", **kw), np.concatenate([s, o], 1))
            assert np.array_equal(m.evaluate(test, corrupt_side="s+o", **kw), s + o - 1)
            assert np.array_equal(m.evaluate(test, corrupt_side="s,o", batch_size=10, **kw),
                                  np.concatenate([s, o], 1))


def test_evaluate_relation_side_ranks_forward_relations_only():
    m, _, t, ent, rel = _trained()
    R = m.max_rel_size
    forward = _model("ComplEx", 16, m.max_ent_size, R, ent, rel[:R], reciprocal=False)
    forward._build_engine()
    forward.is_fitted = True
    test = t[::5]
    for use_filter in (False, {"train": t}):
        for strategy in ("worst", "middle"):
            got = m.evaluate(test, corrupt_side="p", use_filter=use_filter, ranking_strategy=strategy, verbose=False)
            want = forward.evaluate(test, corrupt_side="p", use_filter=use_filter, ranking_strategy=strategy,
                                    verbose=False)
            assert np.array_equal(got, want) and got.max() <= R + 1  # 'worst' counts the positive among the ties


def test_predict_and_embeddings_are_forward():
    m, plain, t, ent, rel = _trained()
    R = m.max_rel_size
    assert np.array_equal(m.predict(t[:50]), plain.predict(t[:50]))
    assert np.array_equal(m.get_embeddings([0, 3], "r"), rel[[0, 3]])
    assert np.array_equal(m.get_embeddings([0, 3], "r_inv"), rel[[R, R + 3]])
    assert np.array_equal(m.get_embeddings([1, 2], "e"), ent[[1, 2]])


# ---------------------------------------------------------------- top-n and discovery
def test_query_topn_head_queries_are_inverse_tail_queries():
    m, plain, t, _, _ = _trained()
    R = m.max_rel_size
    X = t[::11]
    for use_filter in (False, {"train": t}):
        pf = {"train": _inv(t, R)} if use_filter else False
        got = discovery.query_topn_batch(m, X, side="s", top_n=7, use_filter=use_filter)
        want = discovery.query_topn_batch(plain, _inv(X, R), side="o", top_n=7, use_filter=pf)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    for s, p, o in t[:3].tolist():
        got_x, got_s = discovery.query_topn(m, top_n=5, relation=p, tail=o)
        want_x, want_s = discovery.query_topn(plain, top_n=5, head=o, relation=p + R)
        assert np.array_equal(got_s, want_s) and np.array_equal(got_x[:, 0], want_x[:, 2])
        assert (got_x[:, 1] == p).all() and (got_x[:, 2] == o).all()
    # tail queries are untouched; relation queries consider the forward relations only
    got = discovery.query_topn_batch(m, X, side="o", top_n=4)
    want = discovery.query_topn_batch(plain, X, side="o", top_n=4)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    labels, _ = discovery.query_topn_batch(m, X, side="p", top_n=R + 2)
    assert all(v is None or v < R for v in labels.ravel()) and (labels[:, :R] != None).all()  # noqa: E711
    rx, _ = discovery.query_topn(m, top_n=2 * R, head=int(t[0, 0]), tail=int(t[0, 2]))
    assert len(rx) == R and set(int(r) for r in rx[:, 1]) == set(range(R))


def test_discover_facts_runs():
    from ampligraph_b200.discovery import discover_facts
    rng = np.random.default_rng(8)
    names = np.array(["e%d" % i for i in range(30)])
    X = np.stack([names[rng.integers(0, 30, 200)], np.array(["r0", "r1", "r2"])[rng.integers(0, 3, 200)],
                  names[rng.integers(0, 30, 200)]], 1)
    m = ScoringBasedEmbeddingModel(eta=1, k=10, scoring_type="ComplEx", reciprocal_relations=True)
    m.compile(optimizer="adam", loss="multiclass_nll")
    m.fit(X, batch_size=64, epochs=5, verbose=False, one_vs_all="s,o")
    facts, ranks = discover_facts(X, m, top_n=50, strategy="random_uniform", max_candidates=40, target_rel="r1")
    assert len(facts) == len(ranks) and len(facts) > 0  # 30 entities: every candidate's mean rank is <= 50
    assert (facts[:, 1] == "r1").all()
    want = m.evaluate(facts, use_filter={"test": X}, corrupt_side="s,o", verbose=False).mean(1)
    assert np.array_equal(ranks, want)


# ---------------------------------------------------------------- validation inside fit
def test_validation_in_fit_is_evaluate():
    rng = np.random.default_rng(9)
    k, E, R, n = 16, 100, 4, 500
    t = np.stack([rng.integers(0, E, n), rng.integers(0, R, n), rng.integers(0, E, n)], 1).astype(np.int32)
    valid = t[:60]
    K = 2 * k
    m = _model("ComplEx", k, E, R, rng.uniform(-0.3, 0.3, (E, K)).astype(np.float32),
               rng.uniform(-0.3, 0.3, (2 * R, K)).astype(np.float32), optimizer="adam")
    stop = EarlyStopping(monitor="val_mrr", patience=10)
    h = m.fit(t, batch_size=128, epochs=4, verbose=False, one_vs_all="s,o", validation_data=valid, validation_freq=2,
              validation_filter={"train": t}, callbacks=[stop])
    ranks = m.evaluate(valid, use_filter={"train": t}, corrupt_side="s,o", verbose=False)
    from ampligraph_b200.evaluation import mr_score, mrr_score
    assert h.history["val_mrr"][-1] == mrr_score(ranks) and h.history["val_mr"][-1] == mr_score(ranks)
    assert stop.stopped_epoch is None
