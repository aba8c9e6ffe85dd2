"""H100 tests of NSCaching (kge_nscaching_step, DESIGN.md 3.20): the refresh and the draw against the restatement of
tests/nscaching_oracle.py for every model, the filter's empty rows, RotatE's phases, determinism, the caches' hardness,
end-to-end fits, and the C-ABI refusals."""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch

import nscaching_oracle as nsc
from ampligraph_b200 import _lib
from ampligraph_b200.datasets import nscaching_tables
from ampligraph_b200.engine import KGEEngine, NSCache

pytestmark = pytest.mark.gpu

MODELS = ["TransE", "DistMult", "ComplEx", "HolE", "RotatE"]


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a)).cuda().contiguous()


def _triples(rng, E, R, n):
    return np.stack([rng.integers(0, E, n), rng.integers(0, R, n), rng.integers(0, E, n)], 1).astype(np.int32)


def _engine(model, E, R, k, eta, rng):
    eng = KGEEngine(model, k, eta, E, R)
    K = eng.internal_k
    ent = rng.normal(0, 0.5, (E, K)).astype(np.float32)
    rel = rng.normal(0, 0.5, (R, K)).astype(np.float32)
    eng.set_embeddings(ent, rel)
    return eng, ent, rel


def _caches(cache):
    return [x.cpu().numpy().copy() for x in cache.ids], [x.cpu().numpy().copy() for x in cache.count]


def _check_refresh(ids, count, want_ids, want_count, infos, n1):
    """The kernel's rows equal the restatement's, except for swaps between candidates whose float64 keys lie within
    the fp32 error band of the selection cutoff (nsc.key_error_bound on each side of the comparison)."""
    for (side, row), info in infos.items():
        got = list(ids[side][row, :count[side][row]])
        want = list(want_ids[side][row, :want_count[side][row]])
        assert count[side][row] == want_count[side][row], (side, row)
        if got == want:
            continue
        pos = {e: c for c, e in enumerate(info["cand"]) if info["valid"][c]}
        got_c = [pos[e] for e in got]
        assert got_c == sorted(got_c), (side, row)  # ascending c
        key = info["key"]
        order = sorted((c for c in range(len(key)) if info["valid"][c]), key=lambda c: (-key[c], c))
        cut = key[order[n1 - 1]]
        for c in set(got_c) ^ set(info["kept"]):
            assert abs(key[c] - cut) <= nsc.key_error_bound(key[c]) + nsc.key_error_bound(cut), (side, row, c)


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("filtered", [False, True])
@pytest.mark.parametrize("n1,n2", [(1, 1), (5, 3), (50, 50), (200, 312)])
@pytest.mark.parametrize("E", [40, 2000])
def test_refresh_and_draw_equal_the_oracle(model, filtered, n1, n2, E):
    """Three consecutive steps on fixed tables; each step's refresh is compared from the kernel's own caches before it,
    and its draw exactly against the restatement's draw from the kernel's caches after it."""
    rng = np.random.default_rng(zlib.crc32(repr((model, filtered, n1, n2, E)).encode()))
    R, k, eta, n, seed = 3, 8, 3, 60, 11
    t = _triples(rng, E, R, n)
    if E == 40:
        t[:8] = np.stack([np.full(8, 5), np.zeros(8, int), rng.integers(0, E, 8)], 1)  # a repeated (s, p)
    eng, ent, rel = _engine(model, E, R, k, eta, rng)
    tables = nscaching_tables(t, E, R, n, filtered)
    cache = NSCache(tables, n1, n2, eng.device)
    known = set(map(tuple, t.tolist())) if filtered else None
    eng.read_negative_misses()
    for step in range(3):
        pre_ids, pre_count = _caches(cache)
        repl, keep = eng.nscaching_negatives(_dev(t), cache.key_rows, cache.update, cache, seed, step)
        ids, count = _caches(cache)
        want_ids, want_count, infos = nsc.refresh(model, t, tables["key_rows"], tables["update"], ent, rel, pre_ids,
                                                  pre_count, n1, n2, seed, step, known, max_rel_size=R)
        _check_refresh(ids, count, want_ids, want_count, infos, n1)
        w_repl, w_keep, w_miss = nsc.draw(t, tables["key_rows"], ids, count, eta, E, seed, step)
        assert (repl.cpu().numpy() == w_repl).all() and (keep.cpu().numpy() == w_keep).all(), step
        assert eng.read_negative_misses() == w_miss
        if not filtered:
            assert w_miss == 0
    eng.close()


def test_keep_is_the_uniform_side():
    rng = np.random.default_rng(2)
    E, R, eta = 300, 4, 5
    t = _triples(rng, E, R, 500)
    eng, _, _ = _engine("ComplEx", E, R, 8, eta, rng)
    cache = NSCache(nscaching_tables(t, E, R, 500), 5, 5, eng.device)
    _, keep = eng.nscaching_negatives(_dev(t), cache.key_rows, cache.update, cache, 3, 9)
    keep = keep.cpu().numpy().copy()
    _, ukeep = eng.sample_negatives(_dev(t), _uniform_tables(eng), 3, 9)
    assert (keep == ukeep.cpu().numpy()).all()
    eng.close()


def _uniform_tables(eng):
    from ampligraph_b200.engine import NegativeSamplerTables
    return NegativeSamplerTables({}, 1, eng.device)


def test_filter_empties_a_full_row_and_counts_its_misses():
    """(5, 0) has every entity as an object: with the filter its object-side row ends empty, its object corruptions
    fall back to the uniform draw and are all misses; no corruption drawn from a non-empty row is a training triple."""
    rng = np.random.default_rng(4)
    E, R, eta = 40, 3, 4
    t = np.concatenate([np.stack([np.full(E, 5), np.zeros(E, int), np.arange(E)], 1), _triples(rng, E, R, 60)])
    t = t.astype(np.int32)
    eng, _, _ = _engine("DistMult", E, R, 8, eta, rng)
    tables = nscaching_tables(t, E, R, len(t), True)
    cache = NSCache(tables, 10, 20, eng.device)
    eng.read_negative_misses()
    repl, keep = eng.nscaching_negatives(_dev(t), cache.key_rows, cache.update, cache, 1, 0)
    repl, keep = repl.cpu().numpy(), keep.cpu().numpy()
    ids, count = _caches(cache)
    full_row = tables["key_rows"][0, 1]
    assert count[1][full_row] == 0
    known = set(map(tuple, t.tolist()))
    B, misses = len(t), 0
    for r in range(B * eta):
        i, side = r % B, int(keep[r])
        s, p, o = (int(x) for x in t[i])
        n = count[side][tables["key_rows"][i, side]]
        if n == 0:
            misses += 1
        else:
            assert ((s, p, int(repl[r])) if side else (int(repl[r]), p, o)) not in known
    assert misses > 0 and eng.read_negative_misses() == misses
    eng.close()


def test_rotate_refresh_reads_the_current_phases():
    rng = np.random.default_rng(5)
    E, R, eta, n1, n2 = 200, 3, 2, 5, 10
    t = _triples(rng, E, R, 40)
    eng, ent, _ = _engine("RotatE", E, R, 8, eta, rng)
    tables = nscaching_tables(t, E, R, len(t))
    cache = NSCache(tables, n1, n2, eng.device)
    eng.nscaching_negatives(_dev(t), cache.key_rows, cache.update, cache, 7, 0)
    rel = rng.normal(0, 2.0, (R, eng.internal_k)).astype(np.float32)
    eng.set_embeddings(None, rel)
    pre_ids, pre_count = _caches(cache)
    eng.nscaching_negatives(_dev(t), cache.key_rows, cache.update, cache, 7, 1)
    ids, count = _caches(cache)
    want = nsc.refresh("RotatE", t, tables["key_rows"], tables["update"], ent, rel, pre_ids, pre_count, n1, n2, 7, 1,
                       max_rel_size=R)
    _check_refresh(ids, count, *want, n1)
    eng.close()


def _structured(E=200, R=4, n=3000, seed=0):
    """o = (s + 7 (p + 1)) mod E: a learnable graph, split into train and test."""
    rng = np.random.default_rng(seed)
    s = rng.integers(0, E, n)
    p = rng.integers(0, R, n)
    x = np.unique(np.stack([s, p, (s + 7 * (p + 1)) % E], 1), axis=0)
    rng.shuffle(x)
    return x[:-100].astype(np.int32), x[-100:].astype(np.int32)


def _model(model):
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    return ScoringBasedEmbeddingModel(eta=5, k=32, scoring_type=model, seed=3, max_ent_size=200, max_rel_size=4)


def _compile(m, loss="pairwise"):
    from ampligraph_b200.latent_features import optimizers
    m.data_indexer = False
    m.compile(optimizer=optimizers.get("adam", {"learning_rate": 0.01}), loss=loss)


def _fit(model, x, epochs=3, **kw):
    m = _model(model)
    _compile(m, kw.pop("loss", "pairwise"))
    m.fit(x, batch_size=100, epochs=epochs, verbose=False, negative_sampler="nscaching",
          negative_sampler_params={"cache_size": 10, "random_size": 20}, **kw)
    return m


def test_two_fits_are_identical_and_start_from_empty_caches():
    x, _ = _structured()
    firsts = []
    from ampligraph_b200 import engine as engine_mod
    orig = engine_mod.KGEEngine.nscaching_negatives

    def spy(self, triples, key_rows, update, cache, seed=0, step=0):
        firsts.append(sum(int(c.sum()) for c in cache.count))
        return orig(self, triples, key_rows, update, cache, seed, step)
    engine_mod.KGEEngine.nscaching_negatives = spy
    try:
        a = _fit("TransE", x, epochs=2)
        n_steps = len(firsts)
        a.fit(x, batch_size=100, epochs=1, verbose=False, negative_sampler="nscaching")
        b = _fit("TransE", x, epochs=2)
    finally:
        engine_mod.KGEEngine.nscaching_negatives = orig
    assert firsts[0] == 0 and firsts[n_steps] == 0 and firsts[n_steps + n_steps // 2] == 0
    assert firsts[1] > 0
    a2 = _fit("TransE", x, epochs=2)
    for u, v in zip(a2.engine.get_embeddings(), b.engine.get_embeddings()):
        assert torch.equal(u, v)
    assert a2.history.history["loss"] == b.history.history["loss"]


def test_cached_entities_score_higher_than_uniform_ones():
    x, _ = _structured()
    m = _model("DistMult")
    _compile(m)
    m.fit(x, batch_size=100, epochs=10, verbose=False)
    eng = m.engine
    q = x[:300]
    tables = nscaching_tables(q, 200, 4, len(q))
    cache = NSCache(tables, 10, 20, eng.device)
    for step in range(10):
        eng.nscaching_negatives(_dev(q), cache.key_rows, cache.update, cache, 5, step)
    scores = eng.corruption_scores(_dev(q), "o").cpu().numpy()  # [b, E] object-side scores of every entity
    ids, count = _caches(cache)
    cached = [scores[i, ids[1][r, :count[1][r]]].mean() for i, r in enumerate(tables["key_rows"][:, 1])]
    assert np.mean(cached) > scores.mean() + 0.1 * scores.std()


@pytest.mark.parametrize("model", ["TransE", "RotatE", "ComplEx"])
@pytest.mark.parametrize("kind", ["filtered", "user_loss", "focusE"])
def test_fit_end_to_end(model, kind):
    """The loss is finite and decreases, and the filtered test MRR is above twice a random ranking's: a uniformly random
    rank among 200 candidates has an expected reciprocal of H_200 / 200 = 0.029."""
    from ampligraph_b200.evaluation import mrr_score
    x, test = _structured()
    kw = {}
    data = x
    if kind == "filtered":
        kw["filter_negatives"] = True
    elif kind == "user_loss":
        kw["loss"] = lambda p, ng: (ng - p.unsqueeze(0) + 1).clamp(min=0).sum()
    else:
        data = np.concatenate([x, np.random.default_rng(1).random((len(x), 1))], 1)
        kw["focusE"] = True
    m = _fit(model, data, epochs=10, **kw)
    loss = m.history.history["loss"]
    assert np.isfinite(loss).all() and loss[-1] < loss[0]
    ranks = m.evaluate(test, batch_size=100, corrupt_side="s,o", verbose=False,
                       use_filter={"train": x, "test": test})
    assert mrr_score(ranks) > 2 * 0.029, mrr_score(ranks)


def test_c_abi_refusals():
    """Every refusal returns its code without a launch: the outputs and the caches keep their sentinels."""
    eng = KGEEngine("DistMult", 8, 4, 50, 3)
    lib, h, st = eng.lib, eng.h, eng._stream()
    t = _dev(np.array([[1, 0, 2], [3, 1, 4]], np.int32))
    kr = _dev(np.array([[0, 0], [1, 1]], np.int32))
    up = _dev(np.ones((2, 2), np.uint8))
    ne = torch.full((8,), -7, dtype=torch.int32, device="cuda")
    nk = torch.full((8,), 9, dtype=torch.uint8, device="cuda")
    miss = torch.zeros(1, dtype=torch.int64, device="cuda")
    ids = torch.full((2, 4), -3, dtype=torch.int32, device="cuda")
    cnt = torch.zeros(2, dtype=torch.int32, device="cuda")
    fk = _dev(np.array([2, 3], np.int64))
    P = lambda x: C.c_void_p(x.data_ptr()) if x is not None else C.c_void_p(0)

    def ok():
        q = _lib.KgeNSCaching(C.sizeof(_lib.KgeNSCaching), 4, 4)
        q.sub_n_keys = q.obj_n_keys = 2
        q.sub_ids = q.obj_ids = ids.data_ptr()
        q.sub_count = q.obj_count = cnt.data_ptr()
        return q

    def call(q, B=2, ent=eng.ent, t_=t, kr_=kr, up_=up, ne_=ne, nk_=nk):
        return lib.kge_nscaching_step(h, C.byref(q), P(ent), P(eng.rel), P(t_), P(kr_), P(up_), B, 0, 0, P(ne_), P(nk_),
                                      P(miss), st)

    bad = []
    q = ok(); q.struct_size -= 8; bad.append(call(q))
    for n1, n2 in ((0, 4), (4, 0), (-1, 4), (500, 13), (1, 512)):
        q = ok(); q.cache_size, q.random_size = n1, n2; bad.append(call(q))
    q = ok(); q.sub_ids = None; bad.append(call(q))
    q = ok(); q.obj_count = None; bad.append(call(q))
    q = ok(); q.obj_n_keys = 0; bad.append(call(q))
    q = ok(); q.sub_filter_n = -1; bad.append(call(q))
    q = ok(); q.obj_filter_n = 2; q.obj_filter_keys = fk.data_ptr(); bad.append(call(q))
    bad.append(call(ok(), B=-1))
    bad.append(call(ok(), B=2 ** 54))  # eta * B = 2^56
    for name in ("ent", "t_", "kr_", "up_", "ne_", "nk_"):
        bad.append(call(ok(), **{name: None}))
    assert bad == [_lib.KGE_ERR_INVALID_ARGUMENT] * len(bad), bad
    assert lib.kge_nscaching_step(h, None, P(eng.ent), P(eng.rel), P(t), P(kr), P(up), 2, 0, 0, P(ne), P(nk), P(miss),
                                  st) == _lib.KGE_ERR_INVALID_ARGUMENT
    # a pending deferred step (eta * B = 80 >= n_ent: the step buckets and defers)
    eng.forward_backward(_dev(np.tile(np.array([[1, 0, 2]], np.int32), (20, 1))), None, seed=0, step=0, defer=True)
    assert eng._deferred
    pending = call(ok())
    eng.apply_gradients()
    stash = torch.zeros(64 * 8, dtype=torch.float32, device="cuda")
    _lib.check(lib.kge_set_row_stash(h, P(stash), 8))
    sharded = call(ok())
    _lib.check(lib.kge_set_row_stash(h, None, 0))
    torch.cuda.synchronize()
    assert bool((ne == -7).all()) and bool((nk == 9).all()) and bool((ids == -3).all()) and int(cnt.sum()) == 0
    assert sharded == _lib.KGE_ERR_UNSUPPORTED
    assert pending == _lib.KGE_ERR_INVALID_ARGUMENT
    assert call(ok(), B=0) == _lib.KGE_OK and call(ok(), B=0, t_=None, ne_=None, nk_=None) == _lib.KGE_OK
    assert call(ok(), B=2) == _lib.KGE_OK
    torch.cuda.synchronize()
    assert bool((ne != -7).all()) and int(miss) == 0 and int(cnt.min()) >= 1
    eng.close()
