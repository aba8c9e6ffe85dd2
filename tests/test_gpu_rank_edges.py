"""The ranking kernels at the quantisation's edges, against the oracle, bit for bit.

Ranks count quantise(score) = int32(fl(score * 1000)) comparisons (truncated, saturated, NaN -> 0: kgeo_quantise,
restated in tests/test_rank_edges_host.py).  The tables here inject chosen scores (test_rank_edges_host.inject_*):
scores on and one ulp around the bin edges n/1000, scores whose fl(score * 1000) leaves the int32 range, and NaN / inf /
-0 entries in candidate rows, positive rows and query vectors, as a diverged fit leaves behind.  Every ranking path must
count them as the oracle does: rank_mode "auto" (tensor-core filter + exact refine) and "exact", the pair and the tile
kernel, the full table, a window, an unsorted subset, filters, raw counters, the relation side and the row-sharded path.
"""
import numpy as np
import pytest
import torch

import relation_oracle as ro
import test_rank_edges_host as H
from oracle import c_oracle
from test_gpu_shards import _finalize, _rank_counts, _rank_engines, _Shards
from topk_oracle import topk as ref_topk

pytestmark = pytest.mark.gpu

MODELS = H.MODELS
TC_MODELS = ["DistMult", "ComplEx", "HolE"]
STRATEGIES = H.STRATEGIES
K_SMALL, E, B = 8, 700, 160  # 700 candidates: three 256-row tiles, the last one short; 160 queries: two 128-query blocks


def _engine(model, k, E, R, ent, rel, rank_mode):
    from ampligraph_b200.engine import KGEEngine
    eng = KGEEngine(model, k, 1, E, R, rank_mode=rank_mode)
    eng.set_embeddings(ent, rel)
    return eng


def _dev(a):
    return torch.as_tensor(a).cuda().contiguous()


def _values(group):
    return {"edges": H.edge_values, "saturate": H.saturating_values, "nonfinite": H.nonfinite_values}[group]()


def _case(model, group, seed):
    rng = np.random.default_rng(seed)
    nonfinite = group == "nonfinite"
    ent, rel, _ = H.inject_tables(model, K_SMALL, _values(group), E, rng, second=0.25 if nonfinite else 0.0,
                                  poison=nonfinite)
    return rng, ent, rel


def _filters(n_rows, b, rng):
    """CSR filters of entity ids: every row of an injected table is edge-valued, so the filter entries are too"""
    lists = [sorted(set(rng.integers(0, n_rows, 6).tolist())) for _ in range(b)]
    off = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int64)
    return lists, off, np.concatenate([np.asarray(x, np.int32) for x in lists])


def _bits_equal(x, y):
    """fp32 arrays equal bit for bit, any NaN equal to any NaN (the device's NaNs are canonical, C's keep payloads)"""
    x, y = np.asarray(x, np.float32), np.asarray(y, np.float32)
    nan = np.isnan(x) & np.isnan(y)
    return bool(((x.view(np.uint32) == y.view(np.uint32)) | nan).all())


# KGE_B200_RANK_KERNEL=tile swaps the pair kernel of TransE / RotatE for the tile kernel; the bilinear models have one
# exact kernel (kge_rank_dot_kernel), so they run the default only
EDGE_CASES = [(m, g, kern) for m in MODELS for g in ("edges", "saturate", "nonfinite")
              for kern in (("default", "tile") if m in ("TransE", "RotatE") else ("default",))]


@pytest.mark.parametrize("model,group,kernel", EDGE_CASES)
def test_rank_edges_vs_oracle(model, group, kernel, monkeypatch):
    """Both sides, both rank modes, every tie strategy: the full table, a window, an unsorted subset, CSR filters of
    edge-valued rows and the raw counters equal the oracle's ranks (and "auto"'s counters "exact"'s) bit for bit."""
    if kernel == "tile":
        monkeypatch.setenv("KGE_B200_RANK_KERNEL", "tile")
    else:
        monkeypatch.delenv("KGE_B200_RANK_KERNEL", raising=False)
    rng, ent, rel = _case(model, group, 11)
    engs = {m: _engine(model, K_SMALL, E, rel.shape[0], ent, rel, m) for m in ("auto", "exact")}
    sub = rng.permutation(E)[:601].astype(np.int32)  # unsorted subset
    for side in ("s", "o"):
        t = H.inject_triples(E, side, B, rng, poison=group == "nonfinite")
        td = _dev(t)
        lists, off, idx = _filters(E, B, rng)
        for i, f in enumerate(lists):  # the positive's own row in every other list
            if i % 2 == 0:
                f.append(int(t[i, 0 if side == "s" else 2]))
        off = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int64)
        idx = np.concatenate([np.asarray(x, np.int32) for x in lists])
        raw = {}
        for mode, eng in engs.items():
            for strategy in STRATEGIES:
                want = c_oracle.rank_triples(model, side, strategy, ent, rel, t)
                got = eng.rank(td, side, strategy).cpu().numpy()
                assert (got == want).all(), (mode, side, strategy, np.flatnonzero(got != want)[:8])
            want = c_oracle.rank_triples(model, side, "middle", ent, rel, t, start_id=45, n_cand=600)
            got = eng.rank(td, side, "middle", cand_begin=45, n_cand=600).cpu().numpy()
            assert (got == want).all(), (mode, side, "window")
            want = c_oracle.rank_triples(model, side, "worst", ent, rel, t, cand_ids=sub)
            got = eng.rank(td, side, "worst", cand_ids=_dev(sub)).cpu().numpy()
            assert (got == want).all(), (mode, side, "subset")
            want = c_oracle.rank_triples(model, side, "best", ent, rel, t, filters=lists)
            got = eng.rank(td, side, "best", _dev(off), _dev(idx)).cpu().numpy()
            assert (got == want).all(), (mode, side, "filtered")
            cnt = torch.zeros((B, 3), dtype=torch.int32, device="cuda")
            eng.rank(td, side, "worst", _dev(off), _dev(idx), counts=cnt)
            raw[mode] = cnt.cpu().numpy()
            for strategy in STRATEGIES:
                want = c_oracle.rank_triples(model, side, strategy, ent, rel, t, filters=lists)
                assert (H.finalize(raw[mode], strategy) == want).all(), (mode, side, strategy, "counts")
        assert (raw["auto"] == raw["exact"]).all(), side
    for eng in engs.values():
        eng.close()


@pytest.mark.parametrize("model", MODELS)
def test_rank_edges_relation_side(model):
    """Side 'p' (kge_rank_rel.cu): relation rows carrying edge and saturating values (RotatE: random phases), queries
    whose entity rows hold NaN, +inf and -inf; every tie strategy, a window, filters and the raw counters."""
    rng = np.random.default_rng(13)
    k, R = K_SMALL, 300
    K = H.width(model, k)
    ent = np.zeros((8, K), np.float32)
    unit = model not in ("TransE", "RotatE")
    ent[:, 0] = 1.0 if unit else 0.0
    ent[2, 1], ent[3, 1], ent[4, 1] = np.nan, np.inf, -np.inf  # non-finite query rows
    ent[5, 0], ent[6, 0], ent[7, 0] = 2147483.75, np.inf, -0.0
    if model == "RotatE":
        rel = rng.uniform(-3, 3, (R, K)).astype(np.float32)
    else:
        vals = np.concatenate([H.edge_values(), H.saturating_values(), [np.nan, np.inf, -np.inf]]).astype(np.float32)
        rel = np.zeros((R, K), np.float32)
        rel[:, 0] = np.concatenate([vals, rng.choice(vals, R - len(vals))])[rng.permutation(R)]
    b = 150
    t = np.stack([rng.integers(0, 8, b), rng.integers(0, R, b), rng.integers(0, 8, b)], 1).astype(np.int32)
    t[:40, 0] = t[:40, 2] = 0  # clean queries: the relation's own value is the score
    eng = _engine(model, k, 8, R, ent, rel, "auto")
    td = _dev(t)
    lists = [sorted(set(rng.integers(0, R, 5).tolist())) for _ in range(b)]
    off = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int64)
    idx = np.concatenate([np.asarray(x, np.int32) for x in lists])
    for strategy in STRATEGIES:
        want = ro.ranks(model, strategy, ent, rel, t)
        got = eng.rank(td, "p", strategy).cpu().numpy()
        assert (got == want).all(), (strategy, np.flatnonzero(got != want)[:8])
    want = ro.ranks(model, "middle", ent, rel, t, cand_begin=17, n_cand=250)
    assert (eng.rank(td, "p", "middle", cand_begin=17, n_cand=250).cpu().numpy() == want).all()
    cnt = torch.zeros((b, 3), dtype=torch.int32, device="cuda")
    eng.rank(td, "p", "worst", _dev(off), _dev(idx), counts=cnt)
    assert (cnt.cpu().numpy() == ro.counts(model, ent, rel, t, filters=lists)).all()
    eng.close()


@pytest.mark.parametrize("W", [2, 3])
@pytest.mark.parametrize("model", MODELS)
def test_rank_edges_sharded(model, W):
    """kge_rank_sharded over W shards of an injected 1,300-row table (edge, saturating and non-finite values), both
    rank modes (W = 2: 650-row shards, so "auto" runs the tensor-core filter per shard): raw counters summed over ranks
    and finalized once equal the oracle's ranks, unfiltered and filtered with global ids."""
    rng = np.random.default_rng(17 + W)
    n = 1300
    vals = np.concatenate([H.edge_values(), H.saturating_values(), H.nonfinite_values()])
    ent, rel, _ = H.inject_tables(model, K_SMALL, vals, n, rng, poison=True)
    full = _engine(model, K_SMALL, n, rel.shape[0], ent, rel, "exact")
    sh = _Shards(full.ent, n, W, grads=False)
    for mode in ("exact", "auto"):
        ranks = _rank_engines(model, K_SMALL, n, rel.shape[0], rel, W, sh.rps, mode)
        for side in ("s", "o"):
            t = H.inject_triples(n, side, B, rng)
            td = _dev(t)
            lists, off, idx = _filters(n, B, rng)
            plain = _rank_counts(ranks, sh, td, side)
            filt = _rank_counts(ranks, sh, td, side, _dev(off), _dev(idx))
            for strategy in STRATEGIES:
                want = c_oracle.rank_triples(model, side, strategy, ent, rel, t)
                assert (_finalize(ranks[0], plain, strategy) == want).all(), (mode, side, strategy)
                want = c_oracle.rank_triples(model, side, strategy, ent, rel, t, filters=lists)
                assert (_finalize(ranks[0], filt, strategy) == want).all(), (mode, side, strategy, "filtered")
        for e in ranks:
            e.close()
    full.close()


def _bf16(x):
    """fp32 -> the nearest bfloat16 (round to nearest even on the bits), as fp32"""
    b = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    r = ((b + 0x7fff + ((b >> 16) & 1)) & 0xffff0000).astype(np.uint32)
    return r.view(np.float32)


def _band_values(model, qpos):
    """entries v near the edges of the positive's bin (U: qc > qpos, L: qc >= qpos, in accumulator units) whose split
    approximation fl(hi + lo) falls on the other side of the edge than the exact score's quantisation: a filter that
    decided them without the refine would count them wrongly"""
    scale = np.float64(H.hole_scale(K_SMALL)) if model == "HolE" else 1.0
    out = []
    for edge, strict in ((qpos + 1, True), (qpos, False)):
        e = np.float32(edge / 1000.0 / scale)
        v = H.ulps(e, 200)
        hi = _bf16(v)
        lo = _bf16(v - hi)
        a = (hi + lo).astype(np.float32)
        assert ((hi.astype(np.float64) + lo) == a).all()  # fl(hi + lo) is exact here: no accumulation order matters
        q = H.quantise(H.closed_score(model, K_SMALL, v))
        exact = q > qpos if strict else q >= qpos
        out.append(v[exact != (a >= e)])
    return np.concatenate(out)


@pytest.mark.parametrize("model", TC_MODELS)
def test_tc_filter_refines_a_tile_with_a_nan_row(model):
    """A NaN row makes its 256-candidate tile's norm, and so the filter's error bound delta, NaN.  Candidates of that
    tile within delta of the positive's bin edges, whose split approximation lands on the wrong side of the edge, must
    still go to the exact refine: "auto" == "exact" == the oracle."""
    rng = np.random.default_rng(19)
    scale = np.float64(H.hole_scale(K_SMALL)) if model == "HolE" else 1.0
    qpos = 1000
    vp = np.float32(1.0005 / scale)
    assert H.quantise(H.closed_score(model, K_SMALL, vp)) == qpos
    band = _band_values(model, qpos)
    assert len(band) >= 8, len(band)
    band = band[rng.permutation(len(band))[:60]]
    ent, rel, _ = H.inject_tables(model, K_SMALL, np.array([np.float32(5.0 / scale), np.float32(-5.0 / scale)]), E, rng)
    ent[256:256 + len(band), 0] = band  # tile 1 (positions 256..511)
    ent[300, 0] = np.nan
    ent[600, 0] = vp  # the positive, in tile 2
    ent[520:520 + len(band), 0] = band  # the same values in a finite tile
    eng = {m: _engine(model, K_SMALL, E, rel.shape[0], ent, rel, m) for m in ("auto", "exact")}
    for side in ("s", "o"):
        t = np.zeros((B, 3), np.int32)
        t[:, 0 if side == "s" else 2] = 600
        t[:, 2 if side == "s" else 0] = H.ANCHOR
        td = _dev(t)
        for strategy in STRATEGIES:
            want = c_oracle.rank_triples(model, side, strategy, ent, rel, t)
            x = eng["exact"].rank(td, side, strategy).cpu().numpy()
            a = eng["auto"].rank(td, side, strategy).cpu().numpy()
            assert (x == want).all() and (a == want).all(), (side, strategy, a[:4], want[:4])
    for e in eng.values():
        e.close()


@pytest.mark.parametrize("model", TC_MODELS)
def test_tc_filter_nonfinite_overflow_falls_back_to_exact(model):
    """NaN and inf rows, queries and positives send whole tiles to the refine list; with a list of 5 pairs it overflows
    and the gated exact kernel recounts the call: the ranks are still the oracle's, both sides, every strategy."""
    rng, ent, rel = _case(model, "nonfinite", 37)
    from ampligraph_b200.engine import KGEEngine
    eng = KGEEngine(model, K_SMALL, 1, E, rel.shape[0], rank_mode="auto", rank_pair_cap=5)
    eng.set_embeddings(ent, rel)
    for side in ("s", "o"):
        t = H.inject_triples(E, side, B, rng)
        td = _dev(t)
        for strategy in STRATEGIES:
            want = c_oracle.rank_triples(model, side, strategy, ent, rel, t)
            got = eng.rank(td, side, strategy).cpu().numpy()
            assert (got == want).all(), (side, strategy, np.flatnonzero(got != want)[:8])
    eng.close()


@pytest.mark.parametrize("model", TC_MODELS)
def test_tc_filter_dense_saturating_and_poisoned(model):
    """Random k = 200 tables scaled so that the positives' scores straddle +-2.147e6 (where fl(score * 1000) leaves the
    int32 range), with a few NaN- and inf-poisoned rows: "auto" == "exact" == the oracle, both sides, every strategy,
    filtered and unfiltered."""
    rng = np.random.default_rng(23)
    k, R = 200, 5
    K = H.width(model, k)
    ent = rng.uniform(-1, 1, (E, K)).astype(np.float32)
    rel = rng.uniform(-1, 1, (R, K)).astype(np.float32)
    t = np.stack([rng.integers(0, E, B), rng.integers(0, R, B), rng.integers(0, E, B)], 1).astype(np.int32)
    c = (2.147e6 / np.std(c_oracle.score_triples(model, ent, rel, t))) ** (1 / 3)
    ent, rel = (ent * np.float32(c)).astype(np.float32), (rel * np.float32(c)).astype(np.float32)
    sc = c_oracle.score_triples(model, ent, rel, t)
    q = H.quantise(sc)
    assert (q == H.INT_MAX).sum() >= 10 and (q == H.INT_MIN).sum() >= 10 and (np.abs(sc) < 2.1e6).sum() >= 10
    for r, col, v in ((5, 3, np.nan), (290, 0, np.inf), (511, 7, -np.inf), (699, 1, np.nan)):
        ent[r, col] = v
    t[:4, 0] = [5, 290, 511, 699]  # poisoned positives and query vectors
    lists, off, idx = _filters(E, B, rng)
    eng = {m: _engine(model, k, E, R, ent, rel, m) for m in ("auto", "exact")}
    td = _dev(t)
    for side in ("s", "o"):
        for strategy in STRATEGIES:
            want = c_oracle.rank_triples(model, side, strategy, ent, rel, t)
            for m, e in eng.items():
                got = e.rank(td, side, strategy).cpu().numpy()
                assert (got == want).all(), (m, side, strategy, np.flatnonzero(got != want)[:8])
        want = c_oracle.rank_triples(model, side, "worst", ent, rel, t, filters=lists)
        for m, e in eng.items():
            assert (e.rank(td, side, "worst", _dev(off), _dev(idx)).cpu().numpy() == want).all(), (m, side, "filtered")
    for e in eng.values():
        e.close()


def test_tc_filter_probe_on_a_nan_tile():
    """kge_rank_filter_probe with a NaN row present still returns a bound for every pair: NaN for every pair of the NaN
    row's tile (no bound: the filter refines them all), finite and sound (|approx - exact| <= delta) everywhere else."""
    rng = np.random.default_rng(29)
    model, k, R = "ComplEx", 24, 3
    ent = rng.uniform(-0.5, 0.5, (E, 2 * k)).astype(np.float32)
    rel = rng.uniform(-0.5, 0.5, (R, 2 * k)).astype(np.float32)
    ent[300, 5] = np.nan
    t = np.stack([rng.integers(0, 256, B), rng.integers(0, R, B), rng.integers(0, 256, B)], 1).astype(np.int32)
    eng = _engine(model, k, E, R, ent, rel, "auto")
    td = _dev(t)
    for side in ("s", "o"):
        approx, delta = (x.cpu().numpy() for x in eng.rank_filter_probe(td, side))
        exact = eng.corruption_scores(td, side).cpu().numpy()
        assert np.isnan(delta[:, 256:512]).all()
        fin = np.r_[0:256, 512:E]
        d = delta[:, fin].astype(np.float64)
        assert (d > 0).all() and (np.abs(approx[:, fin].astype(np.float64) - exact[:, fin]) <= d).all()
        assert (eng.rank(td, side, "middle").cpu().numpy() == c_oracle.rank_triples(model, side, "middle", ent, rel, t)).all()
    eng.close()


def test_rotate_nonfinite_pair_tile_oracle_and_topk(monkeypatch):
    """RotatE's object-side modulus (the branch-free sqrt of kge_rank_common.cuh) on NaN and +inf: the pair kernel, the
    tile kernel and the oracle give the same corruption scores bit for bit (NaN for a NaN entry, -inf for an infinite
    one), both sides, and top-k puts the NaN candidates first."""
    rng = np.random.default_rng(31)
    model, k, R, n = "RotatE", 40, 4, 777
    ent = rng.uniform(-0.5, 0.5, (n, 2 * k)).astype(np.float32)
    rel = rng.uniform(-3, 3, (R, 2 * k)).astype(np.float32)
    ent[10, 3] = np.nan
    ent[300, k + 7] = np.inf
    ent[301, 0] = -np.inf
    ent[600, 1] = 3e19  # re^2 overflows to +inf
    ent[601, 2] = -0.0
    clean = np.setdiff1d(np.arange(n), [10, 300, 301, 600, 601])  # the other queries' own rows stay finite
    t = np.stack([rng.choice(clean, 90), rng.integers(0, R, 90), rng.choice(clean, 90)], 1).astype(np.int32)
    t[:4, 0] = [10, 300, 600, 601]
    t[4:8, 2] = [10, 300, 600, 601]
    eng = _engine(model, k, n, R, ent, rel, "exact")
    td = _dev(t)
    for side in ("s", "o"):
        want = c_oracle.corruption_scores(model, side, ent[t[:, 0]], rel[t[:, 1]], ent[t[:, 2]], ent, max_rel_size=R)
        assert np.isnan(want[:, 10]).all() and (want[8:, 300] == -np.inf).all() and (want[8:, 600] == -np.inf).all()
        got = {}
        for kern in ("pair", "tile"):
            if kern == "tile":
                monkeypatch.setenv("KGE_B200_RANK_KERNEL", "tile")
            else:
                monkeypatch.delenv("KGE_B200_RANK_KERNEL", raising=False)
            got[kern] = eng.corruption_scores(td, side).cpu().numpy()
            assert _bits_equal(got[kern], want), (side, kern, np.argwhere(~((got[kern] == want) | np.isnan(got[kern]) & np.isnan(want)))[:5])
            for strategy in STRATEGIES:
                r = eng.rank(td, side, strategy).cpu().numpy()
                assert (r == c_oracle.rank_triples(model, side, strategy, ent, rel, t)).all(), (side, kern, strategy)
        ids, scores = (x.cpu().numpy() for x in eng.topk(td, side, 5))
        pos, val = ref_topk(want, 5)
        assert (ids == pos).all() and _bits_equal(scores, val), side
        assert (ids[8:, 0] == 10).all()  # the NaN candidate first
    monkeypatch.delenv("KGE_B200_RANK_KERNEL", raising=False)
    eng.close()
