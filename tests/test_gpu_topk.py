"""GPU tests of top-k link prediction: kge_topk / kge_select_topk (csrc/kge_topk.cu) through the engine, and the
discovery facade (query_topn, query_topn_batch).  Ids and scores must equal the host restatement of the ordering
contract (tests/topk_oracle.py) applied to the oracle's corruption-score matrix, bit for bit."""
import ctypes as C
import logging

import numpy as np
import pytest
import torch

from topk_oracle import topk as ref_topk

pytestmark = pytest.mark.gpu

MODELS = ["TransE", "DistMult", "ComplEx", "HolE", "RotatE"]


def _dev(a):
    return torch.as_tensor(a).cuda().contiguous()


def _tables(model, E, R, k, rng, coarse=False):
    """coarse: entries in {-0.5, 0, 0.5} and the entity rows drawn from 40 distinct ones, so that every model -- RotatE's
    moduli included -- scores many candidates equally."""
    K = k if model in ("TransE", "DistMult") else 2 * k
    if coarse:
        draw = lambda n: rng.choice(np.array([-0.5, 0.0, 0.5], np.float32), (n, K))
        return draw(40)[rng.integers(0, 40, E)], draw(R)
    draw = lambda n: rng.uniform(-0.5, 0.5, (n, K)).astype(np.float32)
    return draw(E), draw(R)


def _triples(E, R, n, rng):
    return np.stack([rng.integers(0, E, n), rng.integers(0, R, n), rng.integers(0, E, n)], 1).astype(np.int32)


def _engine(model, k, E, R, ent, rel, monkeypatch, chunk=None):
    from ampligraph_b200.engine import KGEEngine
    if chunk is None:
        monkeypatch.delenv("KGE_B200_TOPK_CHUNK", raising=False)
    else:
        monkeypatch.setenv("KGE_B200_TOPK_CHUNK", str(chunk))  # read when the handle is created
    eng = KGEEngine(model, k, 1, E, R)
    eng.set_embeddings(ent, rel)
    return eng


def _oracle_scores(model, side, ent, rel, t, R):
    from oracle import c_oracle
    return c_oracle.corruption_scores(model, side, ent[t[:, 0]], rel[t[:, 1]], ent[t[:, 2]], ent, max_rel_size=R)


def _expect(scores, k, exclude=None, to_id=None):
    pos, val = ref_topk(scores, k, exclude)
    ids = pos if to_id is None else np.where(pos >= 0, to_id(np.maximum(pos, 0)), -1)
    return ids, val


def _same(got, want):
    gi, gs = (x.cpu().numpy() for x in got)
    wi, ws = want
    assert gi.shape == wi.shape and (gi == wi).all(), np.argwhere(gi != wi)[:5]
    assert (gs.view(np.uint32) == ws.astype(np.float32).view(np.uint32)).all()


# ---------------------------------------------------------------------------
@pytest.mark.parametrize("chunk", [None, 256])
@pytest.mark.parametrize("model", MODELS)
def test_topk_vs_oracle(model, chunk, monkeypatch):
    """All candidates, a cand_begin/n_cand window and a cand_ids subset (unsorted: position order is not id order), on a
    table whose size is not a multiple of 256, k from 1 to n_cand."""
    rng = np.random.default_rng(11)
    E, R, k, b = 1000, 6, 24, 37
    ent, rel = _tables(model, E, R, k, rng)
    t = _triples(E, R, b, rng)
    eng = _engine(model, k, E, R, ent, rel, monkeypatch, chunk)
    sub = rng.choice(E, 300, replace=False).astype(np.int32)
    for side in ("s", "o"):
        ref = _oracle_scores(model, side, ent, rel, t, R)
        for top in (1, 7, 300, E):
            _same(eng.topk(_dev(t), side, top), _expect(ref, top))
            _same(eng.topk(_dev(t), side, top, cand_begin=100, n_cand=333),
                  _expect(ref[:, 100:433], top, to_id=lambda p: p + 100))
            _same(eng.topk(_dev(t), side, top, cand_ids=_dev(sub)), _expect(ref[:, sub], top, to_id=lambda p: sub[p]))
    eng.close()


@pytest.mark.parametrize("model", MODELS)
def test_topk_ties_independent_of_chunk(model, monkeypatch):
    """Coarse tables give many equal scores: positions break the ties, whatever the chunk."""
    rng = np.random.default_rng(12)
    E, R, k, b = 777, 4, 8, 29
    ent, rel = _tables(model, E, R, k, rng, coarse=True)
    t = _triples(E, R, b, rng)
    for side in ("s", "o"):
        ref = _oracle_scores(model, side, ent, rel, t, R)
        assert len(np.unique(ref[0])) < E // 4  # the point of the test: ties everywhere
        for chunk in (None, 256, 100):
            eng = _engine(model, k, E, R, ent, rel, monkeypatch, chunk)
            for top in (5, 300):
                _same(eng.topk(_dev(t), side, top), _expect(ref, top))
            eng.close()


def test_select_topk_special_values():
    from ampligraph_b200.engine import KGEEngine
    eng = KGEEngine("DistMult", 4, 1, 10, 2)
    rng = np.random.default_rng(13)
    pool = np.array([np.nan, -np.nan, np.inf, -np.inf, 0.0, -0.0, 1.0, -1.0, 2.5, 1e-40, -1e-40], np.float32)
    mats = [pool[rng.integers(0, len(pool), (9, 50))], np.full((3, 70), 0.25, np.float32),
            np.array([[np.nan], [-0.0], [-np.inf]], np.float32), pool[rng.integers(0, len(pool), (2, 5000))],
            rng.standard_normal((4, 9000)).astype(np.float32)]
    mats[0][1] = -0.0
    mats[0][2, ::2] = 0.0
    for m in mats:
        for top in (1, 3, m.shape[1], m.shape[1] + 7):
            _same(eng.select_topk(_dev(m), top), _expect(m, top))
    eng.close()


@pytest.mark.parametrize("chunk", [None, 64])
@pytest.mark.parametrize("model", ["ComplEx", "TransE"])
def test_topk_filters(model, chunk, monkeypatch):
    """Filtered positions never appear; a row whose filter leaves fewer than k candidates is padded with -1 / -inf;
    filter entries outside the candidate window are ignored; with a subset the filter holds subset positions."""
    rng = np.random.default_rng(14)
    E, R, k, b = 600, 5, 12, 16
    ent, rel = _tables(model, E, R, k, rng)
    t = _triples(E, R, b, rng)
    eng = _engine(model, k, E, R, ent, rel, monkeypatch, chunk)
    lo, n = 50, 200
    filt = [rng.choice(E, int(rng.integers(0, 120)), replace=False) for _ in range(b)]
    filt[3] = np.arange(lo, lo + n - 5)  # leaves 5 of the window
    filt[4] = np.arange(0, lo)  # entirely outside the window
    off = np.concatenate([[0], np.cumsum([len(f) for f in filt])]).astype(np.int64)
    idx = np.concatenate(filt).astype(np.int32)
    sub = rng.choice(E, 150, replace=False).astype(np.int32)
    for side in ("s", "o"):
        ref = _oracle_scores(model, side, ent, rel, t, R)
        top = 10
        got = eng.topk(_dev(t), side, top, _dev(off), _dev(idx), cand_begin=lo, n_cand=n)
        want = _expect(ref[:, lo:lo + n], top, [f - lo for f in filt], to_id=lambda p: p + lo)
        _same(got, want)
        ids = got[0].cpu().numpy()
        for i in range(b):
            assert not set(ids[i].tolist()) & set(filt[i].tolist())
        assert (ids[3, 5:] == -1).all() and np.isneginf(got[1].cpu().numpy()[3, 5:]).all()
        # all candidates, full-width k: every unfiltered candidate comes back, the rest is padding
        got = eng.topk(_dev(t), side, E, _dev(off), _dev(idx))
        _same(got, _expect(ref, E, filt))
        # subset: the filter holds subset positions
        spos = [rng.choice(len(sub), 40, replace=False) for _ in range(b)]
        soff = np.concatenate([[0], np.cumsum([len(f) for f in spos])]).astype(np.int64)
        sidx = np.concatenate(spos).astype(np.int32)
        got = eng.topk(_dev(t), side, 30, _dev(soff), _dev(sidx), cand_ids=_dev(sub))
        _same(got, _expect(ref[:, sub], 30, spos, to_id=lambda p: sub[p]))
    eng.close()


@pytest.mark.parametrize("E,k,b,top", [(14505, 200, 1024, 100), (1_000_000, 16, 64, 50)])
def test_topk_scale(E, k, b, top, monkeypatch):
    """ComplEx at the cfg2 size and against a million entities (many L2-sized chunks): equal to a host lexsort of
    corruption_scores for the same queries."""
    rng = np.random.default_rng(15)
    R = 20
    ent, rel = _tables("ComplEx", E, R, k, rng)
    t = _triples(E, R, b, rng)
    eng = _engine("ComplEx", k, E, R, ent, rel, monkeypatch)
    del ent
    for side in ("o", "s"):
        full = eng.corruption_scores(_dev(t), side).cpu().numpy()
        _same(eng.topk(_dev(t), side, top), _expect(full, top))
    eng.close()


def test_topk_errors():
    """k = 0, a short workspace and a misaligned workspace are rejected with ValueError (kge_last_error through
    _lib.check); b = 0 is a no-op."""
    from ampligraph_b200 import _lib
    from ampligraph_b200.engine import KGEEngine, _ptr
    E, R = 300, 3
    eng = KGEEngine("DistMult", 8, 1, E, R)
    t = _dev(np.array([[1, 0, 2], [3, 1, 4]], np.int32))
    with pytest.raises(ValueError, match="k must be"):
        eng.topk(t, "o", 0)
    with pytest.raises(ValueError, match="k must be"):
        eng.select_topk(_dev(np.zeros((2, 5), np.float32)), 0)
    lib = eng.lib
    need = lib.kge_topk_workspace_bytes(eng.h, 2, E, 5)
    assert need > 0
    raw = torch.empty(need + 4096, dtype=torch.uint8, device="cuda")
    base = raw.data_ptr() + (-raw.data_ptr()) % 1024
    ids = torch.empty((2, 5), dtype=torch.int32, device="cuda")
    sc = torch.empty((2, 5), dtype=torch.float32, device="cuda")

    def call(ws, nbytes):
        return lib.kge_topk(eng.h, 1, _ptr(eng.ent), _ptr(eng.rel), _ptr(t), 2, None, 0, E, None, None, 0, 5, _ptr(ids),
                            _ptr(sc), C.c_void_p(ws), nbytes, eng._stream())
    with pytest.raises(ValueError, match="workspace of"):
        _lib.check(call(base, need - 1))
    with pytest.raises(ValueError, match="aligned"):
        _lib.check(call(base + 256, need))
    with pytest.raises(ValueError, match="exceeds n_ent"):
        _lib.check(lib.kge_topk(eng.h, 1, _ptr(eng.ent), _ptr(eng.rel), _ptr(t), 2, None, 10, E, None, None, 0, 5,
                                _ptr(ids), _ptr(sc), C.c_void_p(base), need, eng._stream()))
    _lib.check(call(base, need))
    assert lib.kge_topk(eng.h, 1, None, None, None, 0, None, 0, E, None, None, 0, 5, None, None, None, 0, None) == 0
    eng.close()


# ---------------------------------------------------------------------------
def _kg(E, R, n, seed):
    rng = np.random.default_rng(seed)
    t = np.unique(np.stack([rng.integers(0, E, n), rng.integers(0, R, n), rng.integers(0, E, n)], 1), axis=0)
    return np.stack([np.char.add("e", t[:, 0].astype(str)), np.char.add("r", t[:, 1].astype(str)),
                     np.char.add("e", t[:, 2].astype(str))], 1)


@pytest.fixture(scope="module")
def fitted():
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    X = _kg(80, 6, 600, 21)
    m = ScoringBasedEmbeddingModel(eta=3, k=16, scoring_type="ComplEx", seed=3)
    m.compile(optimizer="adam", loss="pairwise")
    m.fit(X, batch_size=100, epochs=3, verbose=False)
    return m, X


def test_query_topn_exceptions(fitted, caplog):
    from ampligraph_b200.discovery import query_topn
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    m, X = fitted
    h, r, t = X[0]
    unfitted = ScoringBasedEmbeddingModel(eta=1, k=4, scoring_type="TransE")
    with pytest.raises(ValueError, match="not fitted"):
        query_topn(unfitted, head=h, relation=r)
    for kw in ({"head": h}, {"head": h, "relation": r, "tail": t}, {}):
        with pytest.raises(ValueError, match="Exactly one"):
            query_topn(m, **kw)
    with pytest.raises(ValueError, match="Head entity"):
        query_topn(m, head="nope", relation=r)
    with pytest.raises(ValueError, match="Relation"):
        query_topn(m, head=h, relation="nope")
    with pytest.raises(ValueError, match="Tail entity"):
        query_topn(m, relation=r, tail="nope")
    with pytest.raises(ValueError, match="ents_to_consider"):
        query_topn(m, head=h, tail=t, ents_to_consider=[h])
    with pytest.raises(ValueError, match="rels_to_consider"):
        query_topn(m, head=h, relation=r, rels_to_consider=[r])
    with pytest.raises(ValueError, match="list or numpy array"):
        query_topn(m, head=h, relation=r, ents_to_consider=(h, t))
    with pytest.raises(ValueError, match="list or numpy array"):
        query_topn(m, head=h, tail=t, rels_to_consider="r0")
    with pytest.raises(ValueError, match="not been seen"):
        query_topn(m, head=h, relation=r, ents_to_consider=[h, "nope"])
    with pytest.raises(ValueError, match="not been seen"):
        query_topn(m, head=h, tail=t, rels_to_consider=[r, "nope"])
    with caplog.at_level(logging.WARNING, logger="ampligraph_b200.discovery"):
        Xo, So = query_topn(m, top_n=5, head=h, relation=r, ents_to_consider=[h, t])
    assert "less than top_n" in caplog.text and Xo.shape == (2, 3) and So.shape == (2,)


def test_query_topn_matches_predict(fitted):
    """Entity completion: the ids of a sort of model.predict over every completion, scores within 1e-4 relative (the
    ranking chain and predict associate some sums differently, DESIGN.md 3.4).  Relation completion: predict's scores
    bit for bit."""
    from ampligraph_b200.discovery import query_topn
    m, X = fitted
    ents, rels = m.data_indexer.ent_labels, m.data_indexer.rel_labels
    for h, r, t in X[:4]:
        for side in ("o", "s"):
            comp = np.array([[h, r, e] for e in ents] if side == "o" else [[e, r, t] for e in ents])
            pred = m.predict(comp)
            pos, _ = ref_topk(pred[None], 10)
            kw = {"head": h, "relation": r} if side == "o" else {"relation": r, "tail": t}
            Xo, So = query_topn(m, top_n=10, **kw)
            assert (Xo == comp[pos[0]]).all()
            assert np.allclose(So, pred[pos[0]], rtol=1e-4, atol=1e-6)
        comp = np.array([[h, x, t] for x in rels])
        pred = m.predict(comp)
        pos, val = ref_topk(pred[None], 4)
        Xo, So = query_topn(m, top_n=4, head=h, tail=t)
        assert (Xo == comp[pos[0]]).all() and (So.view(np.uint32) == val[0].view(np.uint32)).all()
    sub = list(ents[::3])
    Xo, So = query_topn(m, top_n=6, head=X[0, 0], relation=X[0, 1], ents_to_consider=sub)
    comp = np.array([[X[0, 0], X[0, 1], e] for e in sub])
    pos, _ = ref_topk(m.predict(comp)[None], 6)
    assert (Xo == comp[pos[0]]).all()
    Xo, So = query_topn(m, top_n=1, head=X[0, 0], relation=X[0, 1])
    assert Xo.shape == (3,) and np.ndim(So) == 0  # the reference's np.squeeze


def test_query_topn_batch_filtered(fitted):
    """query_topn_batch with use_filter == query_topn over every entity with the known triples removed, per query."""
    from ampligraph_b200.discovery import query_topn, query_topn_batch
    m, X = fitted
    known = {tuple(x) for x in X}
    Q = X[:40]
    for side in ("o", "s"):
        labels, scores = query_topn_batch(m, Q, side=side, top_n=8, use_filter={"train": X})
        assert labels.shape == (40, 8) and scores.dtype == np.float32
        n_ent = len(m.data_indexer.ent_labels)
        for i, (h, r, t) in enumerate(Q):
            kw = {"head": h, "relation": r} if side == "o" else {"relation": r, "tail": t}
            Xo, So = query_topn(m, top_n=n_ent, **kw)
            keep = [j for j, x in enumerate(Xo) if tuple(x) not in known][:8]
            col = 2 if side == "o" else 0
            assert list(labels[i, :len(keep)]) == [Xo[j][col] for j in keep]
            assert (scores[i, :len(keep)] == So[keep]).all()
            assert all(v is None for v in labels[i, len(keep):])
        # unfiltered: the side column is ignored
        garbage = Q.copy()
        garbage[:, 2 if side == "o" else 0] = "whatever"
        a = query_topn_batch(m, garbage, side=side, top_n=5)
        b = query_topn_batch(m, Q, side=side, top_n=5)
        assert (a[0] == b[0]).all() and (a[1] == b[1]).all()
