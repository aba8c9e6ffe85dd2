"""cfg5's shape on one GPU, on an entity table past 2^31 elements: ComplEx, k = 1000 (row stride 2000 floats), 1,000
relations, self_adversarial (margin 3, alpha 0.5), eta = 50, 1,100,000 entities (2.2e9 floats, 8.8 GB).  Row 536,870
straddles element 2^30 (byte 2^32) and row 1,073,741 element 2^31, so any 32-bit element or byte offset on the paths
below reads or writes the wrong row there.

The table is large_table_oracle's: a pool of 4,093 Glorot rows spread over the entities by an integer hash, with unique
sentinel rows around both boundaries, at both ends and at random high ids, written on the device.  The oracles run on
the source rows and expand their results through the id -> source map, so each case checks against the same chains as
the small-table tests:
  * the initialisers bit for bit (Glorot, uniform, constant) and the Philox corruptions;
  * one training step per element within exact_oracle.TrilinearBound on the compacted subproblem of its touched rows, on
    the general kernel's column windows with its default and explicit negative groups and with the row stash;
  * the dense and the lazy Adam step after it bit for bit against optim_exact_oracle, untouched rows bit-identical to
    the fill, gradients back to 0, the lazy rows' stamps;
  * ranking (exact and tensor-core filter + refine, the overflow fallback), corruption scores, top-k, k-NN and scoring.

Each case holds one engine at a time, prints its peak device memory against its budget (the engine's blocks plus its
workspaces and 1.5 GB of temporaries, within what the benchmark's cfg5 run at 1.25 M entities holds), and shows that
its comparison fails when the kernel's output for a straddling row is replaced by that of the neighbouring row."""
import contextlib
import functools
import gc

import numpy as np
import pytest
import torch

import exact_oracle as xo
import large_table_oracle as lt
import optim_exact_oracle as oo
from oracle import c_oracle, philox
from topk_oracle import topk as ref_topk

pytestmark = pytest.mark.gpu

MODEL, k, K, ETA, R, E = "ComplEx", 1000, 2000, 50, 1000, lt.BIG_E
LOSS, LP = "self_adversarial", {"margin": 3.0, "alpha": 0.5}
LD, KP = 2000, 1000
B0, B1 = lt.BIG_BOUNDARIES  # 536,870 and 1,073,741
SLACK = 1.5e9  # fill chunks, gathers and the step's small buffers
BLOCK = (E + R) * LD * 4  # one [ent | rel] block


WIDE = 0.5  # the ranking cases' value range: Glorot-scaled rows score within one quantisation bin of 0


@functools.lru_cache(maxsize=2)
def _spec(wide=False):
    return lt.make_spec(K, seed=5, lim=WIDE if wide else None)


@functools.lru_cache(maxsize=2)
def _rel(wide=False):
    rng = np.random.default_rng(6)
    lim = WIDE if wide else np.sqrt(6.0 / (R + K))
    return rng.uniform(-lim, lim, (R, K)).astype(np.float32)


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a)).cuda().contiguous()


def _free_or_skip(need, what):
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip("%s needs %.2f GB of device memory; %.2f GB is free" % (what, need / 1e9, free / 1e9))


@contextlib.contextmanager
def big_engine(what, blocks=2, ws=None, wide=False, **kw):
    """A filled engine of cfg5's shape.  blocks: [ent | rel] blocks the engine holds (parameters and gradients, plus
    the optimizer's slots); ws(eng): the workspace bytes the case adds; wide: the ranking cases' tables.  Peak memory
    is asserted against the budget when the case body returns; the engine is closed and its memory released in every
    case."""
    from ampligraph_b200.engine import KGEEngine
    gc.collect()
    torch.cuda.empty_cache()
    _free_or_skip(blocks * BLOCK + SLACK, what)
    torch.cuda.reset_peak_memory_stats()
    kw.setdefault("optimizer", "sgd")
    kw.setdefault("optimizer_params", {"learning_rate": 2.0 ** -6})
    eng = KGEEngine(MODEL, k, ETA, E, R, loss=LOSS, loss_params=LP, **kw)
    try:
        assert (eng.ld, eng.kp, eng.internal_k) == (LD, KP, K)
        extra = int(ws(eng)) if ws is not None else 0
        budget = blocks * BLOCK + extra + SLACK
        _free_or_skip(budget - torch.cuda.memory_allocated(), what + " (workspace)")
        lt.fill(eng.ent, _spec(wide), KP)
        eng.set_embeddings(None, _rel(wide))
        yield eng
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated()
        print("\n%s: peak device memory %.2f GB, budget %.2f GB (blocks %d x %.2f GB, workspace %.2f GB)"
              % (what, peak / 1e9, budget / 1e9, blocks, BLOCK / 1e9, extra / 1e9))
        assert peak <= budget, (what, peak, budget)
    finally:
        eng.close()
        del eng
        gc.collect()
        torch.cuda.empty_cache()


def _ids(rng, n):
    """n ids: the sentinels and ids spread over the table, denser toward its end."""
    spread = (E - 1 - np.floor((E - 1) * rng.random(600) ** 2)).astype(np.int64)
    return rng.choice(np.concatenate([_spec().sentinels, spread]), n)


def _step_inputs(seed, B):
    """Positives (s, o from _ids; the straddling rows and their neighbours among them) and injected negatives."""
    rng = np.random.default_rng(seed)
    t = np.stack([_ids(rng, B), rng.integers(0, R, B), _ids(rng, B)], 1).astype(np.int32)
    t[0, 0], t[1, 2], t[2, 0], t[3, 2] = B1, B0, B1 + 1, B0 + 1
    ne = _ids(rng, ETA * B).astype(np.int32)
    nk = rng.integers(0, 2, ETA * B).astype(np.uint8)
    return t, ne, nk


def _touched(t, ne):
    return np.unique(np.concatenate([t[:, 0], t[:, 2], ne]).astype(np.int64))


# ---------------------------------------------------------------------------
# 1. initialisers and the corruption stream
# ---------------------------------------------------------------------------
def test_initialisers_and_corruptions_bit_exact():
    """Glorot (seed 3: the entity table draws with 6), uniform [-1/4, 3/4) (seed 4 -> 8) and constant on every checked
    row bit for bit against large_table_oracle's restatement of kge_misc.cu's counter layout; the constant over the
    whole table.  generate_corruptions over 3,200 rows against philox.corruption_stream."""
    rng = np.random.default_rng(11)
    rows = np.unique(np.concatenate([[0, B0 - 1, B0, B0 + 1, B1 - 1, B1, B1 + 1, E - 2, E - 1],
                                     rng.integers(B1, E, 12)]))
    with big_engine("initialisers") as eng:
        at = _dev(rows.astype(np.int64))
        eng.init_glorot_uniform(seed=3, only="ent")
        got = eng.ent[at].cpu().numpy()
        want = np.stack([lt.glorot_row(int(r), E, K, 6) for r in rows])
        assert (got.view(np.uint32) == want.view(np.uint32)).all(), rows[(got != want).any(1)]
        i = int(np.flatnonzero(rows == B1)[0])
        assert not (got[i + 1].view(np.uint32) == want[i].view(np.uint32)).all(), "sensitivity: neighbour's row"

        eng.init_table("ent", "uniform", -0.25, 0.75, seed=4)
        got = eng.ent[at].cpu().numpy()
        want = np.stack([lt.uniform_row(int(r), K, -0.25, 0.75, 8) for r in rows])
        assert (got.view(np.uint32) == want.view(np.uint32)).all(), rows[(got != want).any(1)]
        assert not (got[i + 1].view(np.uint32) == want[i].view(np.uint32)).all(), "sensitivity: neighbour's row"

        eng.init_table("ent", "constant", 0.3)
        c = torch.tensor(0.3, dtype=torch.float32).view(torch.int32).cuda()
        for a in range(0, E, 65536):
            assert bool((eng.ent[a:a + 65536].view(torch.int32) == c).all()), a

        t = _step_inputs(12, 64)[0]
        got = eng.generate_corruptions(_dev(t), seed=9, step=1_000_003).cpu().numpy()
        want = philox.corruption_stream(t, ETA, E, 9, 1_000_003)
        assert (got == want).all(), np.argwhere(got != want)[:5]
        repl = np.where(want[:, 0] != np.tile(t[:, 0], ETA), want[:, 0], want[:, 2])
        assert repl.max() > B1  # the replacement ids reach past the second boundary
        print("initialisers: %d rows bit-exact (glorot, uniform), constant over %d rows; %d corruptions"
              % (len(rows), E, len(want)))


# ---------------------------------------------------------------------------
# 2. one training step
# ---------------------------------------------------------------------------
PATHS = {"general": dict(neg_group=0, stash=False), "groups": dict(neg_group=3, stash=False),
         "stash": dict(neg_group=0, stash=True)}


@pytest.mark.parametrize("path", list(PATHS))
def test_training_step_within_bound(path):
    """512 positives, 25,600 injected negatives over the sentinels and ids weighted toward the table's end.  The general
    kernel runs: the fast paths need rows that fit one 512-column window, and a step that does not run them never
    buckets (kge_train_workspace_bytes is 0).  It runs with its default negative groups, with groups of 3, and re-reading
    the replaced rows from the row stash, which the step must have written over its NaN fill.  Scores, loss and every
    element of the touched g_ent / g_rel rows within TrilinearBound of the float64 oracle on the compacted tables; the
    rows with a non-zero gradient are exactly the touched ones, and the table is unchanged.

    The path rests on the library's decision, not on kernel names from torch.profiler: a profiling session around a
    step of this size leaves later sessions in the same process recording no kernels, which the RotatE and trilinear
    tests rely on."""
    B = 512
    cfg = PATHS[path]
    t, ne, nk = _step_inputs(21, B)
    U = _touched(t, ne)
    with big_engine("train %s" % path, neg_group=cfg["neg_group"]) as eng:
        assert eng.lib.kge_rows_resident(eng.h) == 0 and int(eng.lib.kge_train_workspace_bytes(eng.h, B)) == 0
        if cfg["stash"]:
            st = eng.ensure_row_stash(B)
            assert st is not None
            st.fill_(float("nan"))
        sp = torch.full((B,), float("nan"), device="cuda")
        sn = torch.full((ETA * B,), float("nan"), device="cuda")
        eng.forward_backward(_dev(t), (_dev(ne), _dev(nk)), scores_pos=sp, scores_neg=sn)
        loss = eng.read_loss()
        g_ent = eng.g_ent[_dev(U)].cpu().double()
        g_rel = eng.g_rel.cpu().double()
        nz_ent, nz_rel = lt.nonzero_rows(eng.g_ent), lt.nonzero_rows(eng.g_rel)
        changed = lt.mismatched_rows(eng.ent, _spec(), KP)
        sp, sn = sp.cpu().double(), sn.cpu().double()
        if cfg["stash"]:
            written = int(torch.isfinite(st).any(1).sum())
            assert written == st.shape[0], "the step did not write every row of the row stash"
            print("\ntrain stash: %d of %d stash rows written" % (written, st.shape[0]))
    assert np.array_equal(nz_ent, U), (len(nz_ent), len(U))
    assert np.array_equal(nz_rel, np.unique(t[:, 1])), "g_rel rows"
    assert changed.size == 0, changed[:5]

    ent_c = _spec().rows[_spec().src[U]]
    t_c = np.stack([np.searchsorted(U, t[:, 0]), t[:, 1], np.searchsorted(U, t[:, 2])], 1)
    ne_c = np.searchsorted(U, ne)
    ref = xo.oracle_step(MODEL, ent_c, _rel(), t_c, ETA, ne_c, nk, loss=LOSS, loss_params=LP, chunk=128)
    bound = xo.TrilinearBound(MODEL, ent_c, _rel(), t_c, ref, ETA, loss=LOSS, loss_params=LP)
    ratios = {}
    for name, got, want in (("sp", sp, ref.sp), ("sn", sn, ref.sn)):
        ok, ratios[name] = bound.check_scores(got, want, name)
        assert ok, (path, name, ratios[name])
    assert abs(loss - ref.loss) <= bound.loss_err, (loss, ref.loss, bound.loss_err)
    ratios["loss"] = abs(loss - ref.loss) / bound.loss_err
    for name, ok, r in bound.check(g_ent, g_rel, ref.g_ent, ref.g_rel):
        ratios[name] = r
        assert ok, (path, name, r)
    print("train %s: %d touched rows, worst error / bound %s"
          % (path, len(U), {n: round(r, 4) for n, r in ratios.items()}))

    # sensitivity: the straddling row's gradient taken from its neighbour's row
    i, j = np.searchsorted(U, [B1, B1 + 1])
    assert U[i] == B1 and U[j] == B1 + 1
    bad = g_ent.clone()
    bad[i] = g_ent[j]
    assert not all(ok for _, ok, _ in bound.check(bad, g_rel, ref.g_ent, ref.g_rel)), "sensitivity"


# ---------------------------------------------------------------------------
# 3. the optimizer after the step
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("opt", ["lazy_adam", "adam"])
def test_adam_after_step_bit_exact(opt):
    """cfg5's lazy Adam and dense Adam (one launch over the [ent | rel] block of 2.2e9 elements) after one step: the
    touched entity rows, their slots and the whole relation table bit for bit against optim_exact_oracle.update from
    the step's own gradient; untouched rows bit-identical to the fill and their slots 0; the gradients back to 0; the
    lazy step stamps exactly the looked-up rows."""
    B = 512
    params = {"learning_rate": 1e-3}
    t, ne, nk = _step_inputs(31, B)
    U = _touched(t, ne)
    with big_engine("optimizer %s" % opt, blocks=4, optimizer=opt, optimizer_params=params) as eng:
        Ud = _dev(U)
        eng.forward_backward(_dev(t), (_dev(ne), _dev(nk)), step=0)
        assert not eng._deferred
        g = eng.g_ent[Ud].cpu().numpy()
        g_rel = eng.g_rel.cpu().numpy()
        eng.apply_gradients()
        x_new = eng.ent[Ud].cpu().numpy()
        a_new, b_new = (s[Ud].cpu().numpy() for s in eng.slots["ent"])
        rel_new = eng.rel.cpu().numpy()
        ra_new, rb_new = (s.cpu().numpy() for s in eng.slots["rel"])
        changed = lt.mismatched_rows(eng.ent, _spec(), KP)
        slot_rows = [lt.nonzero_rows(s) for s in eng.slots["ent"]]
        g_left = (lt.nonzero_rows(eng.g_ent).size, lt.nonzero_rows(eng.g_rel).size)
        stamps = None
        if opt.startswith("lazy"):
            s = eng.lib.kge_step_stamp(0)
            stamps = [(eng.stamps[key] == s).nonzero().flatten().cpu().numpy() for key in ("ent", "rel")]
            stamps += [int(torch.count_nonzero(eng.stamps[key])) for key in ("ent", "rel")]
    cfg = oo.config("adam", params)
    z = np.zeros_like(g)
    want = oo.update(cfg, 1, _spec().rows[_spec().src[U]], g, z, z)
    for name, got, w in (("x", x_new, want[0]), ("m", a_new, want[1]), ("v", b_new, want[2])):
        assert (oo.bits(got) == oo.bits(w)).all(), (opt, name, U[(oo.bits(got) != oo.bits(w)).any(1)][:5])
    zr = np.zeros_like(g_rel)
    want_r = oo.update(cfg, 1, _rel(), g_rel, zr, zr)
    for name, got, w in (("rel", rel_new, want_r[0]), ("rel m", ra_new, want_r[1]), ("rel v", rb_new, want_r[2])):
        assert (oo.bits(got) == oo.bits(w)).all(), (opt, name)
    assert np.array_equal(changed, U), (opt, "rows changed", len(changed), len(U))
    assert all(np.array_equal(r, U) for r in slot_rows), (opt, "slot rows")
    assert g_left == (0, 0), (opt, "gradients left", g_left)
    if stamps is not None:
        assert np.array_equal(stamps[0], U) and np.array_equal(stamps[1], np.unique(t[:, 1])), "stamped rows"
        assert stamps[2:] == [len(U), len(np.unique(t[:, 1]))], "unstamped rows hold 0"
    print("optimizer %s: %d touched rows bit-exact" % (opt, len(U)))

    i, j = np.searchsorted(U, [B1, B1 + 1])
    bad = x_new.copy()
    bad[i] = x_new[j]
    assert not (oo.bits(bad) == oo.bits(want[0])).all(), "sensitivity"


# ---------------------------------------------------------------------------
# 4. ranking and the all-candidate passes
# ---------------------------------------------------------------------------
def _queries(seed, b):
    rng = np.random.default_rng(seed)
    t = np.stack([_ids(rng, b), rng.integers(0, R, b), _ids(rng, b)], 1).astype(np.int32)
    t[0, 0], t[1, 0], t[2, 2], t[3, 2] = B1, B1 + 1, B0, B0 + 1
    return t, rng


def _filters(t, side, rng):
    """Per query: entries on both straddling rows' neighbourhoods and the query's own id, sorted."""
    near = np.concatenate([np.arange(B0 - 3, B0 + 4), np.arange(B1 - 3, B1 + 4)])
    col = 0 if side == "s" else 2
    lists = [sorted(set(rng.choice(near, 5).tolist()) | {int(q[col])}) for q in t]
    off = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int64)
    return lists, _dev(off), _dev(np.concatenate(lists).astype(np.int32))


def _pos_filters(b, n, rng):
    lists = [sorted(set(rng.integers(0, n, 4).tolist()) | {0, 1}) for _ in range(b)]
    off = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int64)
    return lists, _dev(off), _dev(np.concatenate(lists).astype(np.int32))


@pytest.mark.parametrize("mode,cap", [("exact", 0), ("auto", 0), ("auto", 5)],
                         ids=["exact", "auto", "auto-overflow"])
def test_ranks_bit_exact(mode, cap):
    """64 queries with s or o on the straddling rows, against all 1.1 M entities on both sides: worst / middle / best,
    filters whose entries are the straddling rows, a 2,000-row window across row 1,073,741, an unsorted subset of 5,000
    high ids with position filters.  'auto-overflow' (an undecided-pair list of 5 against blocks of ~270 tied pool rows)
    recounts the call on the exact kernel."""
    b = 64
    t, rng = _queries(41, b)
    td = _dev(t)
    sub = rng.permutation(np.arange(B1 - 20_000, E))[:5000].astype(np.int32)
    sub[:3] = (B1 + 1, B1, B1 - 1)
    win = (B1 - 1000, 2000)
    n_calls = 0
    ws = lambda e: e.lib.kge_rank_workspace_bytes(e.h, b, E)
    with big_engine("rank %s cap=%d" % (mode, cap), rank_mode=mode, rank_pair_cap=cap, ws=ws, wide=True) as eng:
        for side in ("s", "o"):
            for strategy in (("worst", "middle", "best") if not cap else ("middle",)):
                got = eng.rank(td, side, strategy).cpu().numpy()
                want = lt.ranks(MODEL, side, strategy, _spec(True), _rel(True), t)
                assert (got == want).all(), (side, strategy, np.flatnonzero(got != want)[:5])
                n_calls += 1
                if side == "o" and strategy == "worst":  # sensitivity: query 0's rank (s = row 1,073,741), query 1's
                    bad = got.copy()
                    bad[0] = got[1]
                    assert not (bad == want).all(), "sensitivity"
            if cap:
                continue
            lists, off, idx = _filters(t, side, rng)
            got = eng.rank(td, side, "worst", off, idx).cpu().numpy()
            want = lt.ranks(MODEL, side, "worst", _spec(True), _rel(True), t, filters=lists)
            assert (got == want).all(), (side, "filtered")
            got = eng.rank(td, side, "middle", off, idx, cand_begin=win[0], n_cand=win[1]).cpu().numpy()
            want = lt.ranks(MODEL, side, "middle", _spec(True), _rel(True), t, filters=lists, start_id=win[0],
                            n_cand=win[1])
            assert (got == want).all(), (side, "window")
            pl, poff, pidx = _pos_filters(b, len(sub), rng)
            got = eng.rank(td, side, "best", poff, pidx, cand_ids=_dev(sub)).cpu().numpy()
            want = lt.ranks(MODEL, side, "best", _spec(True), _rel(True), t, filters=pl, cand_ids=sub)
            assert (got == want).all(), (side, "subset")
            n_calls += 3
    print("rank %s cap=%d: %d calls bit-exact" % (mode, cap, n_calls))


def test_all_candidate_passes():
    """corruption_scores on a window across row 1,073,741 (bit-exact), top-100 over all 1.1 M entities with blocks of
    tied pool rows (ids and score bits), k-NN with queries on the straddling rows over eng.ent as the points (ids and
    distance bits, both metrics), and score() on triples of sentinel rows (the scoring test's tolerance)."""
    b, win = 64, (B1 - 1000, 2000)
    t, rng = _queries(51, b)
    td = _dev(t)
    qids = np.array([B0, B1, B1 + 3, B1 + 4, E - 1], np.int32)  # B1 + 4 is a pool row: ~270 rows at distance 0
    assert B1 + 4 not in set(_spec(True).sentinels.tolist())

    def ws(e):
        return (e.lib.kge_rank_workspace_bytes(e.h, b, win[1]) + e.lib.kge_topk_workspace_bytes(e.h, 8, E, 100)
                + e.lib.kge_knn_workspace_bytes(e.h, len(qids), E, 64, LD))  # the cached scratch grows: old + new

    sent = _spec(True).sentinels
    st = np.stack([rng.choice(sent, 300), rng.integers(0, R, 300), rng.choice(sent, 300)], 1).astype(np.int32)
    with big_engine("all-candidate passes", ws=ws, wide=True) as eng:
        cs = {side: eng.corruption_scores(td, side, cand_begin=win[0], n_cand=win[1]).cpu().numpy() for side in "so"}
        tk = {side: [x.cpu().numpy() for x in eng.topk(td[:8], side, 100)] for side in "so"}
        nn = {m: [x.cpu().numpy() for x in eng.knn(eng.ent, _dev(qids), 64, m)] for m in ("euclidean", "manhattan")}
        sc = eng.score(_dev(st)).cpu().numpy()
    for side in "so":
        want = lt.corruption_scores(MODEL, side, _spec(True), _rel(True), t, start_id=win[0], n_cand=win[1])
        assert (cs[side].view(np.uint32) == want.view(np.uint32)).all(), side
        bad = cs[side].copy()
        bad[:, B1 - win[0]] = cs[side][:, B1 + 1 - win[0]]
        assert not (bad.view(np.uint32) == want.view(np.uint32)).all(), "sensitivity"

        full = lt.corruption_scores(MODEL, side, _spec(True), _rel(True), t[:8])
        wpos, wval = ref_topk(full, 100)
        ids, vals = tk[side]
        assert (ids == wpos).all() and (vals.view(np.uint32) == wval.view(np.uint32)).all(), side
        assert any(len(np.unique(v)) < 100 for v in vals), "top-k without tied pool rows"
    for m, (ids, d) in nn.items():
        D = lt.distances(m, _spec(True), qids, KP, LD)
        wpos, wval = ref_topk(-D, 64)
        assert (ids == wpos).all() and (d.view(np.uint32) == (-wval).view(np.uint32)).all(), m
        assert (d[3] == 0).all() and (ids[0][0], ids[1][0]) == (B0, B1), m
        bad = ids.copy()
        bad[1] = ids[2]
        assert not (bad == wpos).all(), "sensitivity"
    rows = _spec(True).rows[_spec(True).src]
    es, ep, eo = rows[st[:, 0]], _rel(True)[st[:, 1]], rows[st[:, 2]]
    ref = c_oracle.score_rows(MODEL, es, ep, eo, R)
    assert np.allclose(sc, ref, rtol=1e-4, atol=1e-5), np.abs(sc - ref).max()
    print("all-candidate passes: corruption scores, top-100, k-NN and scores as the oracle")
