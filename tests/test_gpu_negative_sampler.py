"""The negative sampler on the GPU (kge_sample_negatives, DESIGN.md 3.18).

- The kernel equals the Python restatement of tests/negative_sampler_oracle.py exactly (entities, sides, miss count)
  for each sampler with and without the filter, and its uniform mode equals kge_generate_corruptions.
- Filtered output holds no training triple except the counted misses; Bernoulli side frequencies lie in a 5 sigma
  binomial band of t_p / 2^32.
- Every training path trains on the sampler's corruptions exactly as on any injected ones: general, resident,
  bucketed deferred (bit for bit against the float64 oracle on exactly representable tables) and RotatE (within the
  bound of the existing RotatE edge test: its sin / cos / sqrt are not exact).
- fit: a filtered fit on collision-free data gives the default fit's tables; user losses and focusE receive the
  sampler's arrays; the C ABI's refusals."""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch

import exact_oracle as xo
import negative_sampler_oracle as nso
from ampligraph_b200 import _lib
from ampligraph_b200.datasets import negative_sampler_tables
from ampligraph_b200.engine import KGEEngine, NegativeSamplerTables
from test_gpu_exact_training import _force, train_exact

pytestmark = pytest.mark.gpu

SAMPLERS = ["uniform", "bernoulli", "pseudo_typed"]
ATTEMPTS = 10


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a)).cuda().contiguous()


def training_set(rng, E=60, R=6, n=400):
    """Skewed relations: p0 1-N (one subject), p1 N-1 (one object), p2 with a single subject AND a dense object set
    (pseudo-typed subject corruptions of it can only rebuild a training triple: forced misses), the rest uniform;
    relation R - 1 has no triples."""
    t = np.stack([rng.integers(0, E, n), rng.integers(3, R - 1, n), rng.integers(0, E, n)], 1)
    m = n // 8
    t[:m] = np.stack([np.full(m, 7), np.zeros(m, int), rng.integers(0, E, m)], 1)
    t[m:2 * m] = np.stack([rng.integers(0, E, m), np.ones(m, int), np.full(m, 11)], 1)
    t[2 * m:3 * m] = np.stack([np.full(m, 5), np.full(m, 2), rng.integers(0, 12, m)], 1)
    return t.astype(np.int32)


def _sample(eng, t, tables, seed, step):
    repl, keep = eng.sample_negatives(_dev(t), tables, seed, step)
    return repl.cpu().numpy(), keep.cpu().numpy(), eng.read_negative_misses()


@pytest.fixture(scope="module")
def engines():
    cache = {}

    def get(eta, E):
        if (eta, E) not in cache:
            cache[(eta, E)] = KGEEngine("DistMult", 8, eta, E, 6)
        return cache[(eta, E)]
    yield get
    for e in cache.values():
        e.close()


@pytest.mark.parametrize("sampler", SAMPLERS)
@pytest.mark.parametrize("filtered", [False, True])
def test_kernel_equals_oracle(sampler, filtered, engines):
    rng = np.random.default_rng(zlib.crc32(repr((sampler, filtered)).encode()))
    E, R = 60, 6
    train = training_set(rng, E, R)
    host = negative_sampler_tables(train, E, R, sampler, filtered)
    tables = NegativeSamplerTables(host, ATTEMPTS, "cuda")
    total_misses = 0
    for B in (1, 37, 1000):
        t = train[rng.integers(0, len(train), B)]
        for eta in (1, 3, 10):
            eng = engines(eta, E)
            for seed, step in ((0, 0), (2 ** 35 + 17, 2 ** 33 + 5)):
                repl, keep, misses = _sample(eng, t, tables, seed, step)
                want = nso.sample(t, eta, E, seed, step, host["thresholds"], host["pools"],
                                  train if filtered else None, ATTEMPTS)
                where = (sampler, filtered, B, eta, seed, step)
                assert (repl == want[0]).all() and (keep == want[1]).all(), where
                assert misses == want[2], (where, misses, want[2])
                if filtered:  # no known triple among the corruptions except the misses
                    known = set(map(tuple, train.tolist()))
                    corr = nso.corrupted_triples(t, eta, repl, keep)
                    assert sum(tuple(x) in known for x in corr.tolist()) == misses, where
                else:
                    assert misses == 0
                total_misses += misses
    if filtered and sampler == "pseudo_typed":
        assert total_misses > 0  # relation 2's subject corruptions
    if sampler == "uniform" and not filtered:
        assert host == {"thresholds": None, "pools": None, "filter": None}


@pytest.mark.parametrize("attempts", [1, 2, 256])
def test_attempt_limits(attempts, engines):
    """max_attempts at 1 (no re-draw), 2 and 256 (the attempt's 8 bits of the counter)."""
    rng = np.random.default_rng(attempts)
    E, R = 60, 6
    train = training_set(rng, E, R)
    host = negative_sampler_tables(train, E, R, "pseudo_typed", True)
    tables = NegativeSamplerTables(host, attempts, "cuda")
    t = train[rng.integers(0, len(train), 500)]
    repl, keep, misses = _sample(engines(3, E), t, tables, 9, 4)
    want = nso.sample(t, 3, E, 9, 4, host["thresholds"], host["pools"], train, attempts)
    assert (repl == want[0]).all() and (keep == want[1]).all() and misses == want[2]


def test_uniform_mode_equals_generate_corruptions():
    """No tables: attempt 0 is kge_generate_corruptions' draw, at bench.py's shape too."""
    rng = np.random.default_rng(3)
    E, R, B, eta = 14505, 237, 27212, 10
    eng = KGEEngine("ComplEx", 8, eta, E, R)
    t = _dev(np.stack([rng.integers(0, E, B), rng.integers(0, R, B), rng.integers(0, E, B)], 1).astype(np.int32))
    tables = NegativeSamplerTables(negative_sampler_tables(np.zeros((0, 3)), E, R), 1, "cuda")
    for seed, step in ((0, 0), (12345, 77)):
        repl, keep = eng.sample_negatives(t, tables, seed, step)
        corr = eng.generate_corruptions(t, seed, step)
        tiled = t.repeat(eta, 1)
        k = keep.bool()
        assert torch.equal(torch.where(k, tiled[:, 0], repl), corr[:, 0])
        assert torch.equal(torch.where(k, repl, tiled[:, 2]), corr[:, 2])
    assert eng.read_negative_misses() == 0
    eng.close()


def test_bernoulli_side_frequencies():
    """Per relation, the share of replaced subjects lies within 5 sigma of p = t_p / 2^32."""
    rng = np.random.default_rng(4)
    E, R = 60, 6
    train = training_set(rng, E, R, n=4000)
    host = negative_sampler_tables(train, E, R, "bernoulli")
    tables = NegativeSamplerTables(host, 1, "cuda")
    eta = 10
    eng = KGEEngine("DistMult", 8, eta, E, R)
    _, keep = eng.sample_negatives(_dev(train), tables, 21, 1)
    rel = np.tile(train[:, 1], eta)
    subj = keep.cpu().numpy() == 0
    p_all = host["thresholds"].astype(np.float64) / 2.0 ** 32
    assert p_all[0] > 0.9 and p_all[1] < 0.1  # 1-N: mostly subjects; N-1: mostly objects
    for p in range(R - 1):
        n = int((rel == p).sum())
        f = float(subj[rel == p].mean())
        sigma = np.sqrt(p_all[p] * (1 - p_all[p]) / n)
        assert abs(f - p_all[p]) <= 5 * sigma + 1e-12, (p, f, p_all[p], n)
    eng.close()


# ---------------------------------------------------------------------------
# training paths on the sampler's corruptions
# ---------------------------------------------------------------------------
def _sampler_negatives(E, R, t, eta, sampler="pseudo_typed", seed=5, step=2):
    """The sampler's (repl, keep) for the positives t, filtered against t itself."""
    host = negative_sampler_tables(t, E, R, sampler, True)
    eng = KGEEngine("DistMult", 8, eta, E, R)
    repl, keep, _ = _sample(eng, t, NegativeSamplerTables(host, ATTEMPTS, "cuda"), seed, step)
    eng.close()
    want = nso.sample(t, eta, E, seed, step, host["thresholds"], host["pools"], t, ATTEMPTS)
    assert (repl == want[0]).all() and (keep == want[1]).all()
    return repl, keep


@pytest.mark.parametrize("path,model,k,sampler", [("general", "ComplEx", 16, "pseudo_typed"),
                                                  ("general", "TransE", 16, "bernoulli"),
                                                  ("resident", "DistMult", 16, "bernoulli"),
                                                  ("resident", "HolE", 8, "pseudo_typed"),
                                                  ("bucketed", "ComplEx", 16, "pseudo_typed")])
def test_exact_paths_on_sampler_corruptions(path, model, k, sampler, monkeypatch):
    rng = np.random.default_rng(zlib.crc32(repr((path, model)).encode()))
    E, R, B, eta = (400, 7, 600, 8) if path != "bucketed" else (500, 9, 700, 8)
    _force(monkeypatch, kernel="general" if path == "general" else None,
           repl="scatter" if path == "resident" else None)
    t = xo.zipf_triples(E, R, B, rng)
    negatives = _sampler_negatives(E, R, t, eta, sampler)
    facts, _ = train_exact(model, k, eta, E, R, B, "pairwise", rng, triples=t, negatives=negatives)
    assert facts["bucketed"] == (eta * B if path == "bucketed" else 0)


@pytest.mark.parametrize("model,k", [("ComplEx", 16), ("DistMult", 33)])
def test_exact_deferred_step_on_sampler_views(model, k, monkeypatch):
    """The deferred bucketed step (replaced-row sum + SGD in one launch) reading the sampler's device buffers: the
    tables equal x0 - lr g, g the float64 oracle's on the same corruptions."""
    _force(monkeypatch)
    rng = np.random.default_rng(zlib.crc32(model.encode()))
    E, R, B, eta, lr = 500, 9, 1000, 4, 2.0 ** -6
    K = xo.internal_k(model, k)
    ent, rel = xo.grid_table(rng, E, K), xo.grid_table(rng, R, K)
    t = xo.zipf_triples(E, R, B, rng)
    eng = KGEEngine(model, k, eta, E, R, loss="pairwise", loss_params={"margin": 1.0}, optimizer="sgd",
                    optimizer_params={"learning_rate": lr})
    eng.set_embeddings(ent, rel)
    tables = NegativeSamplerTables(negative_sampler_tables(t, E, R, "bernoulli", True), ATTEMPTS, "cuda")
    negs = eng.sample_negatives(_dev(t), tables, 3, 1)
    ne, nk = (x.cpu().numpy() for x in negs)
    launches = eng.launches
    eng.forward_backward(_dev(t), negs, seed=3, step=1, defer=True)
    assert eng._deferred
    eng.apply_gradients()
    assert eng.launches - launches == 5
    ref = xo.oracle_step(model, ent, rel, t, eta, ne, nk, loss="pairwise", loss_params={"margin": 1.0})
    for table, x0, g in ((eng.ent, ent, ref.g_ent), (eng.rel, rel, ref.g_rel)):
        want = torch.as_tensor(x0, dtype=torch.float64) - lr * g.cpu()
        xo.assert_fp32_exact(want)
        got = table.detach().cpu()
        got = got[:, :k].double() if K == k else torch.cat([got[:, :k], got[:, eng.kp:eng.kp + k]], 1).double()
        assert torch.equal(got, want)
    eng.close()


def test_rotate_path_on_sampler_corruptions(monkeypatch):
    """RotatE's fast path on the sampler's corruptions, against the float64 oracle within the bound of
    test_gpu_exact_training's RotatE edge test (sin, cos and sqrt are not exact in fp32)."""
    _force(monkeypatch)
    rng = np.random.default_rng(6)
    E, R, B, eta, k = 300, 5, 400, 6, 16
    ent = xo.dyadic_table(rng, E, 2 * k, frac_bits=2)
    rel = xo.dyadic_table(rng, R, 2 * k, frac_bits=2)
    t = xo.zipf_triples(E, R, B, rng)
    ne, nk = _sampler_negatives(E, R, t, eta, "bernoulli")
    lp = {"margin": 3.0, "alpha": 0.5}
    eng = KGEEngine("RotatE", k, eta, E, R, loss="self_adversarial", loss_params=lp)
    eng.set_embeddings(ent, rel)
    eng.forward_backward(_dev(t), (_dev(ne), _dev(nk)))
    torch.cuda.synchronize()
    ge = torch.cat([eng.g_ent[:, :k], eng.g_ent[:, eng.kp:eng.kp + k]], 1).double().cpu()
    gr = torch.cat([eng.g_rel[:, :k], eng.g_rel[:, eng.kp:eng.kp + k]], 1).double().cpu()
    eng.close()
    ref = xo.oracle_step("RotatE", ent, rel, t, eta, ne, nk, loss="self_adversarial", loss_params=lp)
    tol = 2.0 ** -14 * max(float(ref.g_ent.abs().max()), float(ref.g_rel.abs().max()))
    assert float((ge - ref.g_ent.cpu()).abs().max()) <= tol and float((gr - ref.g_rel.cpu()).abs().max()) <= tol


# ---------------------------------------------------------------------------
# fit
# ---------------------------------------------------------------------------
def _fit_model(x, E, R, k, ent, rel, **fit_kw):
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel, optimizers
    m = ScoringBasedEmbeddingModel(eta=2, k=k, scoring_type="DistMult", seed=7, max_ent_size=E, max_rel_size=R)
    m.data_indexer = False
    m.compile(optimizer=optimizers.get("sgd", {"learning_rate": 2.0 ** -6}), loss="pairwise",
              entity_relation_initializer=[ent, rel])
    m.fit(x, batch_size=len(x), epochs=1, verbose=False, **fit_kw)
    return m


def test_filtered_fit_on_collision_free_data_equals_default_fit():
    """Every corruption this fit draws misses the training set (checked on the host replay), so the filter re-draws
    nothing: the step is the default one, bit for bit on exactly representable tables."""
    rng = np.random.default_rng(8)
    E, R, n, k = 5000, 3, 200, 16
    x = np.stack([rng.integers(0, E, n), rng.integers(0, R, n), rng.integers(0, E, n)], 1).astype(np.int32)
    known = set(map(tuple, x.tolist()))
    corr = _lib.host_corruptions(x, 2, E, seed=7, step=0)
    assert not any(tuple(c) in known for c in corr.tolist())  # the premise: nothing collides
    ent, rel = xo.grid_table(rng, E, k), xo.grid_table(rng, R, k)
    plain = _fit_model(x, E, R, k, ent, rel)
    filt = _fit_model(x, E, R, k, ent, rel, filter_negatives=True)
    assert filt.negative_filter_misses == 0
    for a, b in zip(plain.engine.get_embeddings(), filt.engine.get_embeddings()):
        assert torch.equal(a, b)
    assert plain.engine.launches + 1 == filt.engine.launches  # the sampler's one launch
    assert plain.history.history["loss"] == filt.history.history["loss"]


@pytest.mark.parametrize("kind", ["user_loss", "focusE"])
def test_two_phase_paths_receive_the_sampler_arrays(kind):
    """fit with a user loss or focusE and a sampler: both kernel calls of every step get the sampler's buffers, whose
    content is the restatement's for (seed, step); the misses are counted once per epoch."""
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    rng = np.random.default_rng(9)
    E, R, n, eta = 40, 6, 300, 3
    x = training_set(rng, E, R, n)
    m = ScoringBasedEmbeddingModel(eta=eta, k=8, scoring_type="ComplEx", seed=4, max_ent_size=E, max_rel_size=R)
    m.data_indexer = False
    m.compile(loss=(lambda p, ng: (ng - p.unsqueeze(0)).clamp(min=0).sum()) if kind == "user_loss" else "pairwise")
    m.max_ent_size, m.max_rel_size = E, R
    m._build_engine()
    eng, seen = m.engine, []
    orig = eng.forward_backward

    def spy(triples, negatives=None, **kw):
        seen.append((triples.cpu().numpy(), negatives, negatives[0].cpu().numpy(), negatives[1].cpu().numpy(),
                     kw["step"]))
        return orig(triples, negatives, **kw)
    eng.forward_backward = spy
    data = x if kind == "user_loss" else np.concatenate([x, rng.random((n, 1))], 1)
    m.fit(data, batch_size=100, epochs=2, verbose=False, focusE=kind == "focusE", negative_sampler="pseudo_typed",
          filter_negatives=True)
    assert len(seen) == 2 * 2 * 3  # forward and backward of 3 steps per epoch
    host = negative_sampler_tables(x, E, R, "pseudo_typed", True)
    misses = 0
    for i in range(0, len(seen), 2):
        (t, negs, ne, nk, step), (_, negs2, ne2, nk2, step2) = seen[i], seen[i + 1]
        assert step == step2 and (ne == ne2).all() and (nk == nk2).all()
        assert negs[0].data_ptr() == eng._neg_ent.data_ptr() and negs2[1].data_ptr() == eng._neg_keep.data_ptr()
        want = nso.sample(t, eta, E, m.seed, step, None, host["pools"], x, 10)
        assert (ne == want[0]).all() and (nk == want[1]).all(), step
        misses += want[2]
    assert misses > 0 and m.negative_filter_misses == misses


def test_c_abi_refusals():
    """Refused with KGE_ERR_INVALID_ARGUMENT and nothing launched: the outputs keep their sentinel."""
    eng = KGEEngine("DistMult", 8, 4, 50, 3)
    lib, h, st = eng.lib, eng.h, eng._stream()
    t = _dev(np.array([[1, 0, 2], [3, 1, 4]], np.int32))
    ne = torch.full((8,), -7, dtype=torch.int32, device="cuda")
    nk = torch.full((8,), 9, dtype=torch.uint8, device="cuda")
    miss = torch.zeros(1, dtype=torch.int64, device="cuda")
    ids = _dev(np.arange(3, dtype=np.int32))
    off = _dev(np.array([0, 1, 2, 3], np.int64))
    P = lambda x: C.c_void_p(x.data_ptr()) if x is not None else C.c_void_p(0)

    def call(q, B=2, t_=t, ne_=ne, nk_=nk):
        return lib.kge_sample_negatives(h, C.byref(q), P(t_), B, 0, 0, P(ne_), P(nk_), P(miss), st)

    def ok():
        return _lib.KgeNegativeSampler(C.sizeof(_lib.KgeNegativeSampler), 10)

    bad = []
    q = ok(); q.struct_size -= 8; bad.append(call(q))
    for a in (0, -1, 257):
        q = ok(); q.max_attempts = a; bad.append(call(q))
    q = ok(); q.sub_pool_off = off.data_ptr(); bad.append(call(q))
    q = ok(); q.obj_pool_ids = ids.data_ptr(); bad.append(call(q))
    q = ok(); q.sub_filter_n = -1; bad.append(call(q))
    q = ok(); q.obj_filter_n = 3; q.obj_filter_vals = ids.data_ptr(); bad.append(call(q))
    bad.append(call(ok(), B=-1))
    bad.append(call(ok(), B=2 ** 54))  # eta * B = 2^56
    bad.append(call(ok(), ne_=None))
    bad.append(call(ok(), nk_=None))
    bad.append(call(ok(), t_=None))
    assert bad == [_lib.KGE_ERR_INVALID_ARGUMENT] * len(bad), bad
    assert lib.kge_sample_negatives(h, None, P(t), 2, 0, 0, P(ne), P(nk), P(miss), st) == _lib.KGE_ERR_INVALID_ARGUMENT
    torch.cuda.synchronize()
    assert bool((ne == -7).all()) and bool((nk == 9).all())
    assert call(ok(), B=0) == _lib.KGE_OK and call(ok(), B=0, t_=None, ne_=None, nk_=None) == _lib.KGE_OK
    assert call(ok(), B=2 ** 54 - 1, t_=None) == _lib.KGE_ERR_INVALID_ARGUMENT  # passes the size check, then null triples
    assert call(ok(), B=2) == _lib.KGE_OK
    torch.cuda.synchronize()
    assert bool((ne != -7).all()) and int(miss) == 0
    eng.close()
