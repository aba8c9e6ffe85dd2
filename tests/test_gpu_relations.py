"""GPU tests of relation prediction, the relation side (side 'p') of kge_rank / kge_corruption_scores / kge_topk
(csrc/kge_rank_rel.cu), and of its facade (evaluate(corrupt_side='p'), query_topn_batch(side='p'),
fit(validation_corrupt_side='p')).  Scores must equal the C oracle's canonical triple score of every completed
(s, r, o) bit for bit, and ranks / top-k lists the restatement of tests/relation_oracle.py."""
import ctypes as C

import numpy as np
import pytest
import torch

import relation_oracle as ro
from topk_oracle import topk as ref_topk

pytestmark = pytest.mark.gpu

MODELS = ["TransE", "DistMult", "ComplEx", "HolE", "RotatE"]


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a)).cuda().contiguous()


def _tables(model, E, R, k, rng, coarse=False):
    """coarse: entries are multiples of 1/8 in [-1/2, 1/2], so that many relations of a query quantise equally."""
    K = k if model in ("TransE", "DistMult") else 2 * k
    if coarse:
        draw = lambda n: (rng.integers(-4, 5, (n, K)) / 8).astype(np.float32)
    else:
        draw = lambda n: rng.uniform(-0.5, 0.5, (n, K)).astype(np.float32)
    return draw(E), draw(R)


def _triples(E, R, n, rng):
    return np.stack([rng.integers(0, E, n), rng.integers(0, R, n), rng.integers(0, E, n)], 1).astype(np.int32)


def _engine(model, k, E, R, ent, rel, max_rel_size=None, monkeypatch=None, chunk=None):
    from ampligraph_b200.engine import KGEEngine
    if monkeypatch is not None:
        if chunk is None:
            monkeypatch.delenv("KGE_B200_TOPK_CHUNK", raising=False)
        else:
            monkeypatch.setenv("KGE_B200_TOPK_CHUNK", str(chunk))  # read when the handle is created
    eng = KGEEngine(model, k, 1, E, R, max_rel_size=max_rel_size)
    eng.set_embeddings(ent, rel)
    return eng


def _bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


# ---------------------------------------------------------------------------
@pytest.mark.parametrize("model", MODELS)
def test_scores_vs_oracle(model):
    """k not a multiple of 4 (pad columns); RotatE with max_rel_size != n_rel; every relation, a window and a subset."""
    rng = np.random.default_rng(31)
    E, R, k, b = 300, 75, 13, 70
    mrs = R + 9 if model == "RotatE" else None
    ent, rel = _tables(model, E, R, k, rng)
    t = _triples(E, R, b, rng)
    eng = _engine(model, k, E, R, ent, rel, max_rel_size=mrs)
    sub = rng.choice(R, 20, replace=False).astype(np.int32)
    for kw, cand in (({}, np.arange(R)), ({"cand_begin": 9, "n_cand": 50}, np.arange(9, 59)),
                     ({"cand_ids": _dev(sub)}, sub)):
        got = eng.corruption_scores(_dev(t), "p", **kw).cpu().numpy()
        want = ro.score_grid(model, ent, rel, t, cand, max_rel_size=mrs)
        assert got.shape == want.shape and (_bits(got) == _bits(want)).all(), np.argwhere(_bits(got) != _bits(want))[:5]
    eng.close()


def _filters(t, R, n_cand, rng, positions):
    """Per query: the positive relation (as a candidate position when `positions`), repeats, random entries and
    entries outside the window."""
    out = []
    for i, (_, r, _) in enumerate(t):
        f = list(rng.integers(0, n_cand, rng.integers(0, 5)))
        if not positions:
            f.append(int(r))
            f += [int(r)] * (i % 2)
        f += [-1 - i % 3, R + i % 4, n_cand + 2]
        out.append([int(v) for v in f])
    return out


def _csr(filters):
    off = np.concatenate([[0], np.cumsum([len(f) for f in filters])]).astype(np.int64)
    idx = np.concatenate([np.asarray(f, np.int32) for f in filters]).astype(np.int32)
    return _dev(off), _dev(idx)


@pytest.mark.parametrize("model", MODELS)
def test_ranks_vs_oracle(model):
    """Every strategy, unfiltered and filtered, over all relations, a cand_begin window and a cand_ids subset without
    the positives; coarse tables force quantised ties.  Raw counters over two partitions, finalized once, equal one
    call ('middle' is not additive)."""
    rng = np.random.default_rng(32)
    E, R, k, b = 200, 70, 6, 100
    mrs = R + 3 if model == "RotatE" else None
    ent, rel = _tables(model, E, R, k, rng, coarse=True)
    t = _triples(E, R, b, rng)
    t[:, 1] = rng.integers(0, 40, b)  # positives outside the subset below
    eng = _engine(model, k, E, R, ent, rel, max_rel_size=mrs)
    sub = rng.permutation(np.arange(40, R))[:20].astype(np.int32)
    cases = [({}, dict()), ({"cand_begin": 5, "n_cand": 50}, dict(cand_begin=5, n_cand=50)),
             ({"cand_ids": _dev(sub)}, dict(cand_ids=sub))]
    ties = 0
    for kw, okw in cases:
        n_cand = len(sub) if "cand_ids" in okw else okw.get("n_cand", R)
        filt = _filters(t, R, n_cand, rng, positions="cand_ids" in okw)
        cnt = ro.counts(model, ent, rel, t, None, max_rel_size=mrs, **okw)
        ties += int(cnt[:, 1].sum())
        for strategy in ("worst", "best", "middle"):
            for f in (None, filt):
                got = eng.rank(_dev(t), "p", strategy, *(_csr(f) if f else (None, None)), **kw).cpu().numpy()
                want = ro.ranks(model, strategy, ent, rel, t, f, max_rel_size=mrs, **okw)
                assert (got == want).all(), (strategy, kw.keys(), f is not None, np.argwhere(got != want)[:5])
    assert ties > b  # the point of the coarse tables
    filt = _filters(t, R, R, rng, positions=False)
    off, idx = _csr(filt)
    counts = torch.zeros((b, 3), dtype=torch.int32, device="cuda")
    eng.rank(_dev(t), "p", "middle", off, idx, cand_begin=0, n_cand=33, counts=counts)
    eng.rank(_dev(t), "p", "middle", off, idx, cand_begin=33, n_cand=R - 33, counts=counts)
    assert (counts.cpu().numpy() == ro.counts(model, ent, rel, t, filt, max_rel_size=mrs)).all()
    got = eng.finalize_ranks(counts, "middle").cpu().numpy()
    assert (got == eng.rank(_dev(t), "p", "middle", off, idx).cpu().numpy()).all()
    assert (got == ro.ranks(model, "middle", ent, rel, t, filt, max_rel_size=mrs)).all()
    eng.close()


@pytest.mark.parametrize("chunk", [None, 16])
@pytest.mark.parametrize("model", MODELS)
def test_topk_vs_oracle(model, chunk, monkeypatch):
    """kge_topk on the relation side == a stable sort of the oracle's score grid, with and without filters, over all
    relations, a window and a subset; chunk 16 sweeps many chunks; k > n_cand pads with -1 / -inf."""
    rng = np.random.default_rng(33)
    E, R, k, b = 150, 70, 10, 45
    ent, rel = _tables(model, E, R, k, rng, coarse=True)
    t = _triples(E, R, b, rng)
    eng = _engine(model, k, E, R, ent, rel, monkeypatch=monkeypatch, chunk=chunk)
    sub = rng.choice(R, 25, replace=False).astype(np.int32)
    for kw, cand, shift in (({}, np.arange(R), 0), ({"cand_begin": 7, "n_cand": 40}, np.arange(7, 47), 7),
                            ({"cand_ids": _dev(sub)}, sub, 0)):
        grid = ro.score_grid(model, ent, rel, t, cand)
        filt = _filters(t, R, len(cand), rng, positions="cand_ids" in kw)
        for f in (None, filt):
            excl = None if f is None else [[v - shift for v in fi] for fi in f]
            for top in (1, 9, len(cand), len(cand) + 6):
                ids, sc = (x.cpu().numpy() for x in eng.topk(_dev(t), "p", top, *(_csr(f) if f else (None, None)), **kw))
                pos, val = ref_topk(grid, top, excl)
                want_ids = np.where(pos >= 0, cand[np.maximum(pos, 0)], -1)
                assert (ids == want_ids).all(), (top, kw.keys(), f is not None)
                assert (_bits(sc) == _bits(val)).all()
    eng.close()


def test_refusals():
    """n_cand beyond n_rel, the tensor-core probe, and the sharded entry point on side 'p'."""
    from ampligraph_b200 import _lib
    rng = np.random.default_rng(34)
    E, R, k = 50, 6, 8
    ent, rel = _tables("DistMult", E, R, k, rng)
    eng = _engine("DistMult", k, E, R, ent, rel)
    t = _dev(_triples(E, R, 4, rng))
    with pytest.raises(ValueError, match="exceeds n_rel"):
        eng.rank(t, "p", n_cand=R + 1)
    with pytest.raises(ValueError, match="exceeds n_rel"):
        eng.topk(t, "p", 3, cand_begin=2, n_cand=R - 1)
    with pytest.raises(ValueError, match="exceeds n_rel"):
        eng.corruption_scores(t, "p", cand_begin=R, n_cand=1)
    with pytest.raises(NotImplementedError):
        eng.rank_filter_probe(t, "p")
    sh = _lib.KgeShardMap()
    sh.struct_size, sh.world, sh.rows_per_shard = C.sizeof(_lib.KgeShardMap), 1, E
    sh.ent[0] = eng.ent.data_ptr()
    ws, need = eng.rank_workspace(4, E)
    out = torch.zeros(4, dtype=torch.int32, device="cuda")
    with pytest.raises(ValueError, match="relation side"):
        _lib.check(eng.lib.kge_rank_sharded(eng.h, C.byref(sh), 0, 2, 0, eng.rel.data_ptr(), t.data_ptr(), 4, None, None,
                                            0, out.data_ptr(), None, ws.data_ptr(), need, None))
    eng.close()


def test_scale_fb15k_shape():
    """FB15k-shaped tables (R = 1,345, ComplEx k = 200) with 4,096 queries: ranks equal the oracle's, filtered."""
    rng = np.random.default_rng(35)
    E, R, k, b = 14951, 1345, 200, 4096
    ent, rel = _tables("ComplEx", E, R, k, rng)
    ent *= 0.2
    t = _triples(E, R, b, rng)
    eng = _engine("ComplEx", k, E, R, ent, rel)
    filt = [[int(t[i, 1])] + list(rng.integers(0, R, 3)) for i in range(b)]
    got = eng.rank(_dev(t), "p", "worst", *_csr(filt)).cpu().numpy()
    assert (got == ro.ranks("ComplEx", "worst", ent, rel, t, filt)).all()
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
    X = _kg(60, 9, 700, 41)  # dense enough that many (s, o) pairs hold several relations
    m = ScoringBasedEmbeddingModel(eta=3, k=16, scoring_type="ComplEx", seed=3)
    m.compile(optimizer="adam", loss="pairwise")
    m.fit(X, batch_size=100, epochs=3, verbose=False)
    return m, X


def test_evaluate_relation_side(fitted):
    """evaluate(corrupt_side='p') == the oracle on the model's tables, plus one, for every strategy and filter."""
    m, X = fitted
    ent, rel = (x.cpu().numpy() for x in m.engine.get_embeddings())
    test = X[::5]
    t = m._index(test)
    known = m._index(X)
    by_so = {}
    for s, r, o in known:
        by_so.setdefault((s, o), set()).add(int(r))
    filt = [sorted(by_so.get((s, o), ())) for s, _, o in t]
    assert sum(len(f) > 1 for f in filt) > 0
    for strategy in ("worst", "best", "middle"):
        for use_filter, f in ((False, None), ({"train": X}, filt)):
            got = m.evaluate(test, use_filter=use_filter, corrupt_side="p", ranking_strategy=strategy, verbose=False)
            assert got.shape == (len(test), 1) and got.dtype == np.int32
            assert (got[:, 0] == ro.ranks("ComplEx", strategy, ent, rel, t, f) + 1).all()
    assert (m.evaluate(test, use_filter={"train": X}, corrupt_side="p", verbose=False) >= 1).all()


def test_query_topn_batch_relations(fitted):
    """query_topn_batch(side='p', use_filter) == query_topn(head, None, tail) with the known triples removed: labels
    equal wherever neighbouring scores differ by more than 1e-4 relative (the two score chains associate differently),
    scores within 1e-4; rels_to_consider restricts the candidates; the 'p' column of X is ignored."""
    from ampligraph_b200.discovery import query_topn, query_topn_batch
    m, X = fitted
    known = {tuple(x) for x in X}
    n_rel = len(m.data_indexer.rel_labels)
    Q = X[:30]
    labels, scores = query_topn_batch(m, Q, side="p", top_n=5, use_filter={"train": X})
    assert labels.shape == (30, 5) and scores.dtype == np.float32
    for i, (h, _, t) in enumerate(Q):
        Xo, So = query_topn(m, top_n=n_rel, head=h, tail=t)
        keep = [j for j, x in enumerate(Xo) if tuple(x) not in known][:5]
        want_l, want_s = [Xo[j][1] for j in keep], So[keep]
        n = len(keep)
        assert np.allclose(scores[i, :n], want_s, rtol=1e-4, atol=1e-6)
        for j in range(n):
            gap = lambda a, c: abs(want_s[a] - want_s[c]) > 1e-4 * max(abs(want_s[a]), abs(want_s[c]), 1e-6)
            clear = (j == 0 or gap(j - 1, j)) and (j == n - 1 or gap(j, j + 1))
            if clear:
                assert labels[i, j] == want_l[j], (i, j)
        assert all(v is None for v in labels[i, n:]) and np.isneginf(scores[i, n:]).all()
    garbage = Q.copy()
    garbage[:, 1] = "whatever"
    a, b = query_topn_batch(m, garbage, side="p", top_n=4), query_topn_batch(m, Q, side="p", top_n=4)
    assert (a[0] == b[0]).all() and (a[1] == b[1]).all()
    rels = list(m.data_indexer.rel_labels[::2])
    lab, sc = query_topn_batch(m, Q, side="p", top_n=len(rels) + 2, rels_to_consider=rels)
    assert set(lab[:, :len(rels)].ravel()) <= set(rels) and all(v is None for v in lab[:, len(rels):].ravel())
    with pytest.raises(ValueError, match="not been seen"):
        query_topn_batch(m, Q, side="p", rels_to_consider=["nope"])
    bad = Q.copy()
    bad[0, 0] = "nope"
    with pytest.raises(ValueError, match="not seen"):
        query_topn_batch(m, bad, side="p")


def test_fit_validates_on_relations():
    """fit(validation_corrupt_side='p') logs the val_mrr evaluate gives on the fitted model."""
    from ampligraph_b200.evaluation import mrr_score
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    X = _kg(60, 9, 700, 42)
    val = X[::7]
    m = ScoringBasedEmbeddingModel(eta=2, k=8, scoring_type="DistMult", seed=5)
    m.compile(optimizer="adam", loss="pairwise")
    hist = m.fit(X, batch_size=200, epochs=2, verbose=False, validation_data=val, validation_freq=2,
                 validation_corrupt_side="p", validation_filter={"train": X})
    ranks = m.evaluate(val, use_filter={"train": X}, corrupt_side="p", verbose=False)
    logged = hist.history["val_mrr"][-1]
    assert logged == pytest.approx(mrr_score(ranks), rel=1e-12)
