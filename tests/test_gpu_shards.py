"""The row-sharded training and ranking kernels and the data-parallel optimizers, on ONE GPU, against the oracle.

A kge_shard_map is W device pointers and the kernels find the owner of entity e as e / rows_per_shard; the sharded and
exchange optimizers take arrays of table and gradient pointers.  W separate allocations on one device therefore exercise
everything of these paths but the peer-memory transport (tests/test_gpu_z_multi.py, two GPUs): the shard addressing with a
short or empty last shard, the filter base of sharded ranking, the rank-order gradient sum, the delivery to every replica,
the ent|rel regulariser switch of the exchange kernel, per-shard row stamps and the row stash under a shard map.  One
handle per "rank", as parallel.ShardedTrainer / DataParallelTrainer use.

No call here waits on a cross-rank flag: with world > 1 on one device, rank 0 would wait for a signal that only a later
launch on the same GPU can send.  So there is no kge_peer_barrier, and every kge_optimizer_step_exchange runs with
phases = 0 (no flag pads).
"""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch

import exact_oracle as xo
import optim_exact_oracle

pytestmark = pytest.mark.gpu

MODELS = ["TransE", "DistMult", "ComplEx", "HolE", "RotatE"]
TC_MODELS = ["DistMult", "ComplEx", "HolE"]
STRATEGIES = ["worst", "best", "middle"]
RTOL = 1e-4
FUSED, FORWARD_ONLY, BACKWARD_EXT = 0, 1, 2  # enum kge_step_mode
MODES = {"fused": FUSED, "forward_only": FORWARD_ONLY, "backward_ext": BACKWARD_EXT}
OLD_STAMP = -3  # what every row stamp holds before the step


def _engine(*a, **kw):
    from ampligraph_b200.engine import KGEEngine
    return KGEEngine(*a, **kw)


def _lib():
    from ampligraph_b200 import _lib as lib
    return lib


def _rng(*key):
    return np.random.default_rng(zlib.crc32(repr(key).encode()))


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _dev(a):
    return torch.as_tensor(a).cuda().contiguous()


def _tables(model, E, R, k, rng, scale):
    K = k if model in ("TransE", "DistMult") else 2 * k
    return (rng.uniform(-scale, scale, (E, K)).astype(np.float32), rng.uniform(-scale, scale, (R, K)).astype(np.float32))


def _triples(E, R, n, rng):
    return np.stack([rng.integers(0, E, n), rng.integers(0, R, n), rng.integers(0, E, n)], 1).astype(np.int32)


def _zipf(E, rng):
    """-> draw(n): ids ~ truncated Zipf(1.0) over a random permutation of [0, E).  A few hot entities take most slots, so the
    gradient scatters of a step pile onto a few rows of a few shards."""
    cdf = np.cumsum(1.0 / np.arange(1, E + 1))
    cdf /= cdf[-1]
    perm = rng.permutation(E)
    return lambda n: perm[np.minimum(np.searchsorted(cdf, rng.random(n)), E - 1)].astype(np.int32)


def _zipf_batch(E, R, B, eta, rng):
    """Zipf positives and Zipf injected negatives (ids, keep_subj) in tile order"""
    draw = _zipf(E, rng)
    t = np.stack([draw(B), rng.integers(0, R, B), draw(B)], 1).astype(np.int32)
    return t, (draw(B * eta), rng.integers(0, 2, B * eta).astype(np.uint8))


def _dense(eng, table):
    """padded [rows, ld] (numpy or torch) -> dense [rows, internal_k], by host-side slicing"""
    t = table.detach().cpu().numpy() if torch.is_tensor(table) else np.asarray(table)
    k, kp = eng.k, eng.kp
    if eng.internal_k == k:
        return t[:, :k].copy()
    return np.concatenate([t[:, :k], t[:, kp:kp + k]], axis=1)


def _close(a, b, rtol=RTOL):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    scale = max(np.abs(b).max(), 1e-30)
    return np.abs(a - b).max() <= rtol * scale + 1e-7


def _bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


class _Shards:
    """A packed [E, ld] entity table (eng.ent after set_embeddings) cut into W separate [rps, ld] allocations on cuda:0,
    the last ones zero-padded, with zeroed gradient shards, optional int32 row-stamp shards (all `stamps`) and the
    kge_shard_map over them -- what W ranks' peer-mapped shards look like to the kernels."""

    def __init__(self, table, E, W, rps=None, grads=True, stamps=None):
        lib = _lib()
        self.E, self.W = E, W
        self.rps = rps = rps or -(-E // W)
        assert rps * W >= E
        full = torch.zeros((rps * W, table.shape[1]), dtype=torch.float32, device="cuda")
        full[:E] = table[:E]
        self.ent = [full[q * rps:(q + 1) * rps].clone() for q in range(W)]
        self.grad = [torch.zeros_like(x) for x in self.ent] if grads else None
        self.stamp = None
        if stamps is not None:
            self.stamp = [torch.full((rps,), int(stamps), dtype=torch.int32, device="cuda") for _ in range(W)]
        self.map = lib.KgeShardMap(C.sizeof(lib.KgeShardMap), W, rps)
        for q in range(W):
            self.map.ent[q] = self.ent[q].data_ptr()
            self.map.grad_ent[q] = self.grad[q].data_ptr() if grads else None
            self.map.stamp_ent[q] = self.stamp[q].data_ptr() if self.stamp is not None else None

    def rows(self, parts):
        """per-shard tensors -> the global [E, ...] view"""
        return torch.cat(parts)[:self.E]


def _slices(B, W):
    b = np.linspace(0, B, W + 1).astype(int)
    return list(zip(b[:-1], b[1:]))


def _tile_slice(a, eta, lo, hi):
    """the rows of a tile-ordered [eta*B, ...] array (row j*B + i) that belong to positives [lo, hi), in the tile order of
    that slice"""
    a = np.asarray(a)
    return np.ascontiguousarray(a.reshape(eta, -1, *a.shape[1:])[:, lo:hi].reshape(-1, *a.shape[1:]))


def _step(engines, mode, t, negs, dpos, dneg, seed, step, sh=None):
    """One step of the global batch t in len(engines) slices of positives, slice r launched through engines[r] (a handle may
    repeat).  sh: train on that shard map (kge_train_step_sharded, every rank into the same gradient shards); None: on each
    engine's own table (kge_train_step).  -> (scores_pos [B], scores_neg [eta*B] in tile order), NaN where not written."""
    lib = _lib()
    eta, B = engines[0].eta, len(t)
    sp = np.full(B, np.nan, np.float32)
    sn = np.full((eta, B), np.nan, np.float32)
    for r, (lo, hi) in enumerate(_slices(B, len(engines))):
        eng, b = engines[r], int(hi - lo)
        if b == 0:
            continue
        td = _dev(t[lo:hi])
        ne = nk = dp = dn = None
        if negs is not None:
            ne, nk = _dev(_tile_slice(negs[0], eta, lo, hi)), _dev(_tile_slice(negs[1], eta, lo, hi))
        if mode == BACKWARD_EXT:
            dp, dn = _dev(dpos[lo:hi]), _dev(_tile_slice(dneg, eta, lo, hi))
        spd = torch.full((b,), float("nan"), device="cuda")
        snd = torch.full((eta * b,), float("nan"), device="cuda")
        out_p, out_n = (None, None) if mode == BACKWARD_EXT else (spd, snd)
        g_rel = None if mode == FORWARD_ONLY else eng.g_rel
        tail = (_ptr(td), b, _ptr(ne), _ptr(nk), seed, step, _ptr(eng.loss_acc), _ptr(out_p), _ptr(out_n), _ptr(dp),
                _ptr(dn), eng._stream())
        if sh is None:
            g_ent = None if mode == FORWARD_ONLY else eng.g_ent
            rc = eng.lib.kge_train_step(eng.h, mode, _ptr(eng.ent), _ptr(eng.rel), _ptr(g_ent), _ptr(g_rel), *tail)
        else:
            rc = eng.lib.kge_train_step_sharded(eng.h, mode, C.byref(sh.map), _ptr(eng.rel), _ptr(g_rel), *tail)
        lib.check(rc)
        sp[lo:hi] = spd.cpu().numpy()
        sn[:, lo:hi] = snd.cpu().numpy().reshape(eta, b)
    return sp, sn.reshape(-1)


# ---------------------------------------------------------------------------------------------------------------------
# kge_train_step_sharded
# ---------------------------------------------------------------------------------------------------------------------
GEOMS = {  # name: model, k, eta, loss, loss parameters, table scale, row stash
    "complex_resident": ("ComplEx", 40, 6, "self_adversarial", {}, 0.3, False),
    "distmult_resident": ("DistMult", 24, 5, "nll", {}, 0.3, False),
    # under a map of W > 1 RotatE takes the general kernel, not kge_train_rot_kernel
    "rotate": ("RotatE", 24, 5, "self_adversarial", {}, 0.3, False),
    "distmult_groups": ("DistMult", 300, 40, "pairwise", {}, 0.2, False),
    "distmult_groups_stash": ("DistMult", 300, 40, "pairwise", {}, 0.2, True),
    "complex_windows": ("ComplEx", 600, 5, "multiclass_nll", {}, 0.05, False),
    # k = 36 is not a power of two: HolE's 2 / k is inexact
    "hole_resident": ("HolE", 36, 6, "nll", {}, 0.3, False),
    # scores near -6 and differences of a few units: margin 2 leaves hinges on both sides of 0, none within its bound
    "transe_resident": ("TransE", 24, 5, "pairwise", {"margin": 2.0}, 0.3, False),
}
NON_RESIDENT = ("distmult_groups", "distmult_groups_stash", "complex_windows")
# (E, W, rows_per_shard): last shard short (1001 = 2*501-1 = 3*334-1 = 8*126-7), 50 rows in 8 shards of 10, whose last
# three hold no rows at all, and a one-rank map (the unsharded kernels through map->ent[0] / map->grad_ent[0])
LAYOUTS = [(1001, 1, None), (1001, 2, None), (1001, 3, None), (1001, 8, None), (50, 8, 10)]
TRAIN_CASES = ([(g, L, "fused", "injected") for g in GEOMS for L in LAYOUTS] +
               [(g, (1001, 3, None), m, "injected") for g in ("complex_resident", "rotate", "distmult_groups_stash",
                                                              "complex_windows") for m in ("forward_only", "backward_ext")] +
               [(g, L, "fused", "philox") for g in ("complex_resident", "rotate", "distmult_groups_stash")
                for L in ((1001, 3, None), (1001, 8, None))])


def _train_kernel(model, geom, W):
    """The fused kernel a step under a W-rank map runs: the general kernel for W > 1 and with a row stash; a one-rank map
    runs the unsharded kernels -- RotatE's fast path, and the resident trilinear fast path for the DistMult, ComplEx
    and HolE geometries whose rows are resident (TransE has none)."""
    if W > 1 or GEOMS[geom][-1]:
        return "kge_train_kernel<"
    if model == "RotatE":
        return "kge_train_rot_kernel<"
    return "kge_train_res_kernel<" if model in xo.TRILINEAR and geom not in NON_RESIDENT else "kge_train_kernel<"


@pytest.mark.parametrize("geom,layout,mode,negatives", TRAIN_CASES,
                         ids=["%s-E%d-W%d-%s-%s" % (g, L[0], L[1], m, n) for g, L, m, n in TRAIN_CASES])
def test_train_step_sharded(geom, layout, mode, negatives, monkeypatch):
    """kge_train_step_sharded over W shards on one device, the batch in W per-rank slices, each launched through its own
    handle into the same gradient shards.  Against the float64 oracle on the dense table: the scores, the loss, every
    element of g_ent (gathered from the shards) and of g_rel (summed over the ranks in float64) within
    exact_oracle.TrilinearBound (RotatE: RotatEBound), with the worst error / bound printed.  Against the unsharded step
    on the same slices (the general kernel for W > 1; the same kernel for W = 1): scores bit-equal, loss within 1e-6,
    gradients within summation-order noise.  The row stamps of every shard and the padding rows of the last ones
    exactly.  Sensitivity: the check rejects the kernels' gradients against the oracle with one corruption's
    dL/dscore multiplied by 1 + 2^-10, the corruption's replaced entity in the last shard that holds rows, with at most
    32 lookups in the step (RotatE, whose bound is looser, and where every replaced entity of that shard has more
    lookups: without the corruption of fewest lookups)."""
    from oracle import c_oracle
    lib = _lib()
    model, k, eta, loss, lp, scale, stash = GEOMS[geom]
    E, W, rps = layout
    R, B, seed, step = 7, 300, 11, 5
    rng = _rng(geom, layout, mode, negatives)
    ent, rel = _tables(model, E, R, k, rng, scale)
    t, negs = _zipf_batch(E, R, B, eta, rng)
    if negatives == "philox":
        negs = None
    dpos = rng.uniform(-1, 1, B).astype(np.float32)
    dneg = rng.uniform(-1, 1, B * eta).astype(np.float32)
    m = MODES[mode]
    where = "%s E=%d W=%d %s %s" % (geom, E, W, mode, negatives)

    # the unsharded step on the same slices
    if W > 1:
        monkeypatch.setenv("KGE_B200_TRAIN_KERNEL", "general")
    ref = _engine(model, k, eta, E, R, loss=loss, loss_params=lp)
    ref.set_embeddings(ent, rel)
    r_sp, r_sn = _step([ref] * W, m, t, negs, dpos, dneg, seed, step)
    torch.cuda.synchronize()
    monkeypatch.delenv("KGE_B200_TRAIN_KERNEL", raising=False)

    sh = _Shards(ref.ent, E, W, rps, grads=mode != "forward_only", stamps=OLD_STAMP)
    ranks = [_engine(model, k, eta, E, R, loss=loss, loss_params=lp, ent_rows=sh.rps) for _ in range(W)]
    for eng in ranks:
        eng.set_embeddings(None, rel)
        if stash:
            assert eng.ensure_row_stash(B) is not None
    assert ref.lib.kge_rows_resident(ranks[0].h) == (0 if geom in NON_RESIDENT else 1)
    out = {}
    names = xo.launched(lambda: out.update(zip(("sp", "sn"), _step(ranks, m, t, negs, dpos, dneg, seed, step, sh=sh))))
    sp, sn = out["sp"], out["sn"]
    torch.cuda.synchronize()

    if negatives == "philox":  # the library's host replay of each slice's draw, in the global tile order
        parts = [lib.host_corruptions(t[lo:hi], eta, E, seed=seed, step=step).reshape(eta, hi - lo, 3)
                 for lo, hi in _slices(B, W)]
        corr = np.concatenate(parts, axis=1).reshape(-1, 3)
    else:
        corr = c_oracle.corrupt(t, eta, negs[1], negs[0])

    # against the unsharded step
    loss_got = sum(float(e.loss_acc[0]) for e in ranks)
    loss_ref = float(ref.loss_acc[0])
    assert abs(loss_got - loss_ref) <= 1e-6 * abs(loss_ref), where
    if mode != "backward_ext":
        assert (sp.view(np.uint32) == r_sp.view(np.uint32)).all() and (sn.view(np.uint32) == r_sn.view(np.uint32)).all()
    if mode != "forward_only":
        g_e = sh.rows(sh.grad)
        g_r = ranks[0].g_rel.double()
        for e in ranks[1:]:
            g_r += e.g_rel.double()
        assert (torch.cat(sh.grad)[E:] == 0).all(), where  # padding rows of the last shards
        assert _close(g_e.cpu().numpy(), ref.g_ent.cpu().numpy(), rtol=2e-5), where
        assert _close(g_r.cpu().numpy(), ref.g_rel.cpu().numpy(), rtol=2e-5), where
    else:
        assert loss_got == 0.0 and all(bool((e.g_rel == 0).all()) for e in ranks)

    # row stamps: exactly the rows of {s, o, replaced ids}, in the shard that owns them
    want = np.full(W * sh.rps, OLD_STAMP, np.int32)
    if mode != "forward_only":
        want[np.unique(np.concatenate([t[:, 0], t[:, 2], corr[:, 0], corr[:, 2]]))] = ref.lib.kge_step_stamp(step)
    assert (torch.cat(sh.stamp).cpu().numpy() == want).all(), where

    # against the float64 oracle on the dense table, element by element
    ext = dict(dpos=dpos, dneg=dneg) if mode == "backward_ext" else {}
    eloss = None if ext else loss
    rot = dict(rot_table=True) if model == "RotatE" else {}
    ora = xo.oracle_step(model, ent, rel, t, eta, corr, None, loss=loss, loss_params=lp, **rot, **ext)
    if model == "RotatE":
        bound = xo.RotatEBound(ent, rel, t, ora, eta, loss=eloss, loss_params=lp)
    else:
        bound = xo.TrilinearBound(model, ent, rel, t, ora, eta, loss=eloss, loss_params=lp)
    ratios = {}
    if mode != "backward_ext":
        for name, got, w in (("sp", sp, ora.sp), ("sn", sn, ora.sn)):
            ok, ratios[name] = bound.check_scores(torch.as_tensor(got, dtype=torch.float64), w, name)
            assert ok, (where, name, "worst error / bound %.3g" % ratios[name])
    if mode == "fused":
        assert abs(loss_got - ora.loss) <= bound.loss_err, (where, loss_got, ora.loss, bound.loss_err)
        ratios["loss"] = abs(loss_got - ora.loss) / bound.loss_err
    if mode != "forward_only":
        (d_e, pads_e), (d_r, pads_r) = xo.dense(ref, g_e), xo.dense(ref, g_r)
        assert pads_e and pads_r, where + ": pad columns written"
        for name, ok, ratio in bound.check(d_e, d_r, ora.g_ent, ora.g_rel):
            ratios[name] = ratio
            if not ok:
                diff = ((d_e - ora.g_ent) if name == "g_ent" else (d_r - ora.g_rel)).abs()
                row = int(diff.max(1).values.argmax())
                raise AssertionError("%s: %s worst error / bound %.3g; largest error in row %d (shard %d)" % (
                    where, name, ratio, row, row // sh.rps if name == "g_ent" else -1))
        # sensitivity: one corruption of the last shard that holds rows, dL/dscore times 1 + 2^-10 (RotatE: dropped,
        # RotatEBound's rule; also where every replaced entity of that shard has more than 32 lookups, as 12,000
        # corruptions over 50 rows have)
        own = np.arange((E - 1) // sh.rps * sh.rps, E)
        pick = None if model == "RotatE" else xo.perturbed_term(model, ent, rel, t, ora, eta, 2.0 ** -10, entities=own)
        if pick is None:
            pick = xo.perturbed_term(model, ent, rel, t, ora, eta, -1.0, entities=own, max_lookups=None, **rot)
        r, one = pick
        res = bound.check(d_e, d_r, ora.g_ent + one.g_ent, ora.g_rel + one.g_rel)
        assert not all(ok for _, ok, _ in res), where + ": the check accepts corruption %d perturbed" % r
    print("\n%s: worst error / bound %s" % (where, {n: round(v, 4) for n, v in ratios.items()}))

    # the kernel that ran (a short profiling session now and then records none: replay the scores into scratch)
    fused = _train_kernel(model, geom, W)
    for _ in range(5):
        if any(fused in n for n in names):
            break
        names |= xo.launched(lambda: _step(ranks, FORWARD_ONLY, t, negs, None, None, seed, step, sh=sh))
    if names:
        assert any(fused in n for n in names), (where, sorted(names))
    else:
        print("%s: the profiler recorded no kernel in six sessions" % where)
    for e in ranks + [ref]:
        e.close()


@pytest.mark.parametrize("model,k,eta,neg_group", [("ComplEx", 40, 6, 0),   # kge_train_res_kernel
                                                   ("RotatE", 24, 5, 0),    # kge_train_rot_kernel
                                                   ("DistMult", 24, 5, 2)])  # kge_train_kernel (negative groups)
def test_one_rank_shard_map_stamps_rows(model, k, eta, neg_group):
    """A one-rank map (a one-process row-sharded run) runs the unsharded kernels, and they must stamp the MAP's row stamps:
    the handle has none of its own (parallel.ShardedTrainer keeps the stamps beside the shards), so without them the lazy
    optimizer would update no entity row at all.  Then one lazy SGD update moves exactly the stamped rows."""
    lib = _lib()
    rng = _rng(model, k, eta)
    E, R, B, step, lr = 1000, 5, 50, 7, 0.1
    ent, rel = _tables(model, E, R, k, rng, 0.3)
    t, negs = _zipf_batch(E, R, B, eta, rng)
    eng = _engine(model, k, eta, E, R, loss="self_adversarial", optimizer="sgd", optimizer_params={"learning_rate": lr},
                  neg_group=neg_group)
    assert eng.stamps["ent"] is None  # dense optimizer: the handle registers no stamps
    eng.set_embeddings(ent, rel)
    sh = _Shards(eng.ent, E, 1, stamps=OLD_STAMP)
    _step([eng], FUSED, t, negs, None, None, 0, step, sh=sh)
    stamp = eng.lib.kge_step_stamp(step)
    touched = np.zeros(E, bool)
    touched[t[:, 0]] = touched[t[:, 2]] = touched[negs[0]] = True
    got = sh.stamp[0].cpu().numpy()
    assert (got[touched] == stamp).all() and (got[~touched] == OLD_STAMP).all()
    x0, g = sh.ent[0].clone(), sh.grad[0].clone()
    lib.check(eng.lib.kge_optimizer_step_lazy(eng.h, C.byref(eng.opt_cfgs["ent"]), 1, _ptr(sh.ent[0]), _ptr(sh.grad[0]), None,
                                              None, E, _ptr(sh.stamp[0]), stamp, None, eng._stream()))
    torch.cuda.synchronize()
    moved = (sh.ent[0] != x0).any(1).cpu().numpy()
    assert (moved == touched).all()
    # the lazy SGD rule, bit for bit: every stamped row x = fma(-g, lr, x), every other row unchanged
    x0n, gn = x0.cpu().numpy(), g.cpu().numpy()
    new, _, _ = optim_exact_oracle.update(eng.opt_cfgs["ent"], 1, x0n, gn, np.zeros_like(x0n), np.zeros_like(x0n))
    want = np.where(touched[:, None], new, x0n)
    assert (optim_exact_oracle.bits(sh.ent[0].cpu().numpy()) == optim_exact_oracle.bits(want)).all()
    assert (sh.grad[0] == 0).all()
    eng.close()


@pytest.mark.parametrize("W", [1, 3])
@pytest.mark.parametrize("model,k,eta", [("ComplEx", 40, 6), ("RotatE", 24, 5)])
def test_lazy_optimizer_over_shards(model, k, eta, W):
    """Three steps of the row-sharded lazy rule, as parallel.ShardedTrainer runs it: kge_train_step_sharded (every rank's
    slice), kge_optimizer_step_lazy on each shard with that shard's stamps, kge_optimizer_step_sharded for the replicated
    relations.  Against RefStep(optimizer="lazy_adam") on the full batch; untouched entity rows are bit-unchanged.  W = 1
    runs the unsharded kernels through a one-rank map."""
    from ampligraph_b200.parallel import row_shard
    from oracle import c_oracle, ref_step
    lib = _lib()
    rng = _rng(model, k, eta, W)
    E, R, B, lr = 1001, 5, 40, 0.01
    ent, rel = _tables(model, E, R, k, rng, 0.3)
    kw = dict(loss="self_adversarial", optimizer="adam", optimizer_params={"learning_rate": lr})
    packer = _engine(model, k, eta, E, R, **kw)
    packer.set_embeddings(ent, rel)
    sh = _Shards(packer.ent, E, W, stamps=0)
    ranks = [_engine(model, k, eta, E, R, ent_rows=sh.rps, **kw) for _ in range(W)]
    for e in ranks:
        e.set_embeddings(None, rel)
    ld = ranks[0].ld
    slots_e = [(torch.zeros_like(x), torch.zeros_like(x)) for x in sh.ent]
    rel_rows = [row_shard(R, W, r) for r in range(W)]
    slots_r = [tuple(torch.zeros((max(hi - lo, 1), ld), device="cuda") for _ in range(2)) for lo, hi in rel_rows]
    rel_ptrs = (C.c_void_p * W)(*[e.rel.data_ptr() for e in ranks])
    grel_ptrs = (C.c_void_p * W)(*[e.g_rel.data_ptr() for e in ranks])
    rs = ref_step.RefStep(model, ent.shape[1], ent, rel, eta, loss="self_adversarial", optimizer="lazy_adam",
                          optimizer_params={"learning_rate": lr})
    touched = np.zeros(E, bool)
    for step in range(3):
        t, negs = _zipf_batch(E, R, B, eta, rng)
        t[:R, 1] = np.arange(R)  # every relation in every step: the dense relation update then equals the lazy one
        _step(ranks, FUSED, t, negs, None, None, 0, step, sh=sh)
        for r, e in enumerate(ranks):
            lib.check(e.lib.kge_optimizer_step_lazy(e.h, C.byref(e.opt_cfgs["ent"]), step + 1, _ptr(sh.ent[r]), _ptr(sh.grad[r]),
                                                    _ptr(slots_e[r][0]), _ptr(slots_e[r][1]), sh.rps, _ptr(sh.stamp[r]),
                                                    e.lib.kge_step_stamp(step), None, e._stream()))
        for r, e in enumerate(ranks):
            lo, hi = rel_rows[r]
            lib.check(e.lib.kge_optimizer_step_sharded(e.h, C.byref(e.opt_cfgs["rel"]), step + 1, W, r, rel_ptrs, grel_ptrs,
                                                       _ptr(slots_r[r][0]), _ptr(slots_r[r][1]), lo, hi, None, e._stream()))
        for e in ranks:
            e.g_rel.zero_()
        rs.train_step(t, c_oracle.corrupt(t, eta, negs[1], negs[0]))
        touched[t[:, 0]] = touched[t[:, 2]] = touched[negs[0]] = True
        assert all(bool((g == 0).all()) for g in sh.grad)  # the lazy update zeroed every gradient row it consumed
    torch.cuda.synchronize()
    got = _dense(packer, sh.rows(sh.ent))
    assert _close(got, rs.ent.detach().numpy(), rtol=5e-4), np.abs(got - rs.ent.detach().numpy()).max()
    assert all(_bits_equal(e.rel, ranks[0].rel) for e in ranks)
    assert _close(_dense(packer, ranks[0].rel), rs.rel.detach().numpy(), rtol=5e-4)
    assert (~touched).sum() > 100 and (got[~touched] == ent[~touched]).all()
    assert (got[touched] != ent[touched]).any(axis=1).all()  # every touched row moved
    assert (torch.cat(sh.ent)[E:] == 0).all()
    for e in ranks + [packer]:
        e.close()


# ---------------------------------------------------------------------------------------------------------------------
# kge_rank_sharded
# ---------------------------------------------------------------------------------------------------------------------
def _rank_engines(model, k, E, R, rel, W, rps, rank_mode="exact"):
    ranks = [_engine(model, k, 1, E, R, ent_rows=rps, rank_mode=rank_mode) for _ in range(W)]
    for e in ranks:
        e.set_embeddings(None, rel)
    return ranks


def _rank_counts(ranks, sh, td, side, off=None, idx=None):
    """every rank's raw counters {greater, equal, filtered} against its own shard: a list of [b, 3] int32"""
    lib = _lib()
    b = td.shape[0]
    n_filt = int(idx.numel()) if idx is not None else 0
    out = []
    for r, e in enumerate(ranks):
        cnt = torch.zeros((b, 3), dtype=torch.int32, device="cuda")
        ws, ws_bytes = e.rank_workspace(b, sh.rps)
        lib.check(e.lib.kge_rank_sharded(e.h, C.byref(sh.map), r, lib.SIDES[side], 0, _ptr(e.rel), _ptr(td), b, _ptr(off),
                                         _ptr(idx), n_filt, None, _ptr(cnt), _ptr(ws), ws_bytes, e._stream()))
        out.append(cnt)
    return out


def _finalize(eng, parts, strategy):
    """sum the raw counters over ranks and apply the tie strategy once"""
    total = parts[0].clone()
    for p in parts[1:]:
        total += p
    return eng.finalize_ranks(total, strategy).cpu().numpy()


def _shard_filters(E, rps, W, own, rng):
    """filter lists of GLOBAL ids spread over every shard that holds rows (the short last one included), with the
    positive's own entity in every other list and the last entity in every fifth"""
    lists = []
    for i, e in enumerate(own):
        ids = {int(rng.integers(q * rps, min((q + 1) * rps, E))) for q in range(W) if q * rps < E and rng.random() < 0.8}
        if i % 2 == 0:
            ids.add(int(e))
        if i % 5 == 0:
            ids.add(E - 1)
        lists.append(sorted(ids))
    off = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int64)
    idx = np.concatenate([np.asarray(x, np.int32) for x in lists]).astype(np.int32)
    return lists, _dev(off), _dev(idx)


def _rank_case(model, k, E, R, b, rng, decimals, scale=0.5):
    ent, rel = _tables(model, E, R, k, rng, scale)
    ent, rel = np.round(ent, decimals), np.round(rel, decimals)  # coarse values: many exact ties
    t = _triples(E, R, b, rng)
    t[0, 0] = t[1, 2] = E - 1
    return ent, rel, t


@pytest.mark.parametrize("W", [2, 3, 8])
@pytest.mark.parametrize("k", [6, 50])
@pytest.mark.parametrize("model", MODELS)
def test_rank_sharded_vs_oracle(model, k, W):
    """kge_rank_sharded over W shards of a 1,001-row table (short last shard), raw counters summed over ranks and finalized
    once: bit for bit the oracle's ranks, both sides, every tie strategy, unfiltered and filtered with global ids."""
    from oracle import c_oracle
    rng = _rng(model, k, W)
    E, R, b = 1001, 6, 64
    ent, rel, t = _rank_case(model, k, E, R, b, rng, 1 if k == 6 else 2)
    full = _engine(model, k, 1, E, R, rank_mode="exact")
    full.set_embeddings(ent, rel)
    sh = _Shards(full.ent, E, W, grads=False)
    t[2, 0] = t[2, 2] = (W - 1) * sh.rps  # first row of the last shard
    ranks = _rank_engines(model, k, E, R, rel, W, sh.rps)
    td = _dev(t)
    for side in ("s", "o"):
        lists, off, idx = _shard_filters(E, sh.rps, W, t[:, 0 if side == "s" else 2], rng)
        plain = _rank_counts(ranks, sh, td, side)
        filt = _rank_counts(ranks, sh, td, side, off, idx)
        for strategy in STRATEGIES:
            got = _finalize(ranks[0], plain, strategy)
            assert (got == c_oracle.rank_triples(model, side, strategy, ent, rel, t)).all(), (side, strategy)
            gotf = _finalize(ranks[0], filt, strategy)
            want = c_oracle.rank_triples(model, side, strategy, ent, rel, t, filters=lists)
            assert (gotf == want).all(), (side, strategy, "filtered", np.flatnonzero(gotf != want)[:5])
            assert (gotf < got).any()  # the filters do remove candidates
    for e in ranks + [full]:
        e.close()


@pytest.mark.parametrize("model", TC_MODELS)
def test_rank_sharded_tensor_core_filter(model):
    """rank_mode="auto" on shards of 1,500 rows: the tensor-core filter runs per shard, and the counters equal "exact"'s and
    the ranks the oracle's, bit for bit."""
    from oracle import c_oracle
    rng = _rng(model, "tc")
    E, R, k, b, W = 3000, 7, 24, 96, 2
    ent, rel, t = _rank_case(model, k, E, R, b, rng, 1, scale=0.6)
    full = _engine(model, k, 1, E, R, rank_mode="exact")
    full.set_embeddings(ent, rel)
    sh = _Shards(full.ent, E, W, grads=False)
    auto = _rank_engines(model, k, E, R, rel, W, sh.rps, "auto")
    exact = _rank_engines(model, k, E, R, rel, W, sh.rps, "exact")
    # the workspace of an "auto" shard holds the tensor-core operand tiles: the filter applies to every shard
    ws_bytes = full.lib.kge_rank_workspace_bytes
    assert ws_bytes(auto[0].h, b, E - sh.rps) > ws_bytes(exact[0].h, b, E - sh.rps)
    td = _dev(t)
    for side in ("s", "o"):
        lists, off, idx = _shard_filters(E, sh.rps, W, t[:, 0 if side == "s" else 2], rng)
        for f in (None, lists):
            o_, i_ = (off, idx) if f else (None, None)
            pa, px = _rank_counts(auto, sh, td, side, o_, i_), _rank_counts(exact, sh, td, side, o_, i_)
            assert all(torch.equal(a, x) for a, x in zip(pa, px)), side
            for strategy in STRATEGIES:
                want = c_oracle.rank_triples(model, side, strategy, ent, rel, t, filters=f)
                assert (_finalize(auto[0], pa, strategy) == want).all(), (side, strategy, f is not None)
    for e in auto + exact + [full]:
        e.close()


@pytest.mark.parametrize("model", ["ComplEx", "TransE"])
def test_rank_sharded_empty_trailing_shards(model):
    """50 rows in 8 shards of 10: ranks 5..7 own no rows and add nothing; the sum is still the oracle's ranks."""
    from oracle import c_oracle
    rng = _rng(model, "empty")
    E, W, rps, R, k, b = 50, 8, 10, 4, 8, 40
    ent, rel, t = _rank_case(model, k, E, R, b, rng, 1)
    full = _engine(model, k, 1, E, R, rank_mode="exact")
    full.set_embeddings(ent, rel)
    sh = _Shards(full.ent, E, W, rps, grads=False)
    ranks = _rank_engines(model, k, E, R, rel, W, rps)
    td = _dev(t)
    for side in ("s", "o"):
        lists, off, idx = _shard_filters(E, rps, W, t[:, 0 if side == "s" else 2], rng)
        for f in (None, lists):
            parts = _rank_counts(ranks, sh, td, side, *((off, idx) if f else ()))
            assert all(bool((p == 0).all()) for p in parts[5:])
            for strategy in STRATEGIES:
                want = c_oracle.rank_triples(model, side, strategy, ent, rel, t, filters=f)
                assert (_finalize(ranks[0], parts, strategy) == want).all(), (side, strategy, f is not None)
    for e in ranks + [full]:
        e.close()


@pytest.mark.parametrize("model", MODELS)
def test_rank_sharded_one_rank_equals_rank(model):
    """A one-rank map: kge_rank_sharded + kge_rank_finalize == kge_rank on the same table, bit for bit, and == the oracle."""
    from oracle import c_oracle
    rng = _rng(model, "one")
    E, R, k, b = 500, 5, 16, 48
    ent, rel, t = _rank_case(model, k, E, R, b, rng, 2)
    eng = _engine(model, k, 1, E, R, rank_mode="exact")
    eng.set_embeddings(ent, rel)
    sh = _Shards(eng.ent, E, 1, grads=False)
    td = _dev(t)
    for side in ("s", "o"):
        lists, off, idx = _shard_filters(E, E, 1, t[:, 0 if side == "s" else 2], rng)
        parts = _rank_counts([eng], sh, td, side, off, idx)
        for strategy in STRATEGIES:
            got = _finalize(eng, parts, strategy)
            assert (got == eng.rank(td, side, strategy, off, idx).cpu().numpy()).all(), (side, strategy)
            assert (got == c_oracle.rank_triples(model, side, strategy, ent, rel, t, filters=lists)).all(), (side, strategy)
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# kge_optimizer_step_sharded and kge_optimizer_step_exchange
# ---------------------------------------------------------------------------------------------------------------------
OPTS = {"sgd": ("sgd", {"learning_rate": 0.05}), "sgd_momentum": ("sgd", {"learning_rate": 0.05, "momentum": 0.9}),
        "adam": ("adam", {"learning_rate": 0.01}), "adagrad": ("adagrad", {"learning_rate": 0.1})}


def _opt_slots(name, params, rows, ld):
    z = lambda v=0.0: torch.full((max(rows, 1), ld), v, dtype=torch.float32, device="cuda")
    if name == "adam":
        return [z(), z()]
    if name == "adagrad":
        return [z(0.1), None]  # initial_accumulator_value
    return [z(), None] if params.get("momentum") else [None, None]


def _packed(rows, ld, k, rng, scale):
    """[rows, ld] with the pad columns zero"""
    x = np.zeros((rows, ld), np.float32)
    x[:, :k] = rng.uniform(-scale, scale, (rows, k))
    return x


def _rank_order_sum(gs):
    """((g0 + g1) + g2) ... in fp32, the order both kernels sum in"""
    acc = gs[0].copy()
    for g in gs[1:]:
        acc = acc + g
    assert acc.dtype == np.float32
    return acc


def _check_replicas(tables, plain, slots, pslots, bounds):
    """every replica bit-identical, equal to kge_optimizer_step on the rank-order sum, slot shards = the plain slots"""
    assert all(_bits_equal(x, tables[0]) for x in tables[1:])
    assert _bits_equal(tables[0], plain)
    for j in (0, 1):
        if pslots[j] is not None:
            assert _bits_equal(torch.cat([slots[r][j][:hi - lo] for r, (lo, hi) in enumerate(bounds)]), pslots[j]), j


@pytest.mark.parametrize("W", [2, 3, 8])
@pytest.mark.parametrize("opt", list(OPTS))
def test_optimizer_step_sharded(opt, W):
    """kge_optimizer_step_sharded with W replica tables and W gradient tables, rank r = 0..W-1 in turn over its rows
    (parallel.row_shard): replicas bit-identical and bit-equal to kge_optimizer_step on the fp32 rank-order sum (both run
    update4), within 1e-5 of the legacy optimizer restatement; gradients read, not changed; regulariser loss summed over
    ranks == lambda * sum |x|^2 of the table before the step."""
    from ampligraph_b200.parallel import row_shard
    from oracle import ref_step
    lib = _lib()
    name, params = OPTS[opt]
    rng = _rng(opt, W, "sharded")
    rows, k, lam = 101, 10, 1e-3
    eng = _engine("DistMult", k, 1, 8, rows, optimizer=name, optimizer_params=params, regularizer={"p": 2, "lambda": lam})
    cfg, ld = eng.opt_cfgs["rel"], eng.ld
    x0 = _packed(rows, ld, k, rng, 0.5)
    tables, plain = [_dev(x0) for _ in range(W)], _dev(x0)
    bounds = [row_shard(rows, W, r) for r in range(W)]
    slots, pslots = [_opt_slots(name, params, hi - lo, ld) for lo, hi in bounds], _opt_slots(name, params, rows, ld)
    tp = (C.c_void_p * W)(*[x.data_ptr() for x in tables])
    ref, xr = ref_step.LegacyOptimizer(name, **params), torch.as_tensor(x0.copy())
    for t in (1, 2):
        gs = [_packed(rows, ld, k, rng, 1.0) for _ in range(W)]
        grads = [_dev(g) for g in gs]
        gp = (C.c_void_p * W)(*[g.data_ptr() for g in grads])
        pre = tables[0].cpu().numpy().astype(np.float64)
        reg = torch.zeros(W, dtype=torch.float64, device="cuda")
        for r, (lo, hi) in enumerate(bounds):
            lib.check(eng.lib.kge_optimizer_step_sharded(eng.h, C.byref(cfg), t, W, r, tp, gp, _ptr(slots[r][0]), _ptr(slots[r][1]),
                                                         lo, hi, C.c_void_p(reg.data_ptr() + 8 * r), eng._stream()))
        gsum = _rank_order_sum(gs)
        gsum_d = _dev(gsum)
        lib.check(eng.lib.kge_optimizer_step(eng.h, C.byref(cfg), t, _ptr(plain), _ptr(gsum_d), _ptr(pslots[0]), _ptr(pslots[1]),
                                             rows, None, eng._stream()))
        torch.cuda.synchronize()
        _check_replicas(tables, plain, slots, pslots, bounds)
        assert all((gd.cpu().numpy() == g).all() for gd, g in zip(grads, gs))
        want = lam * (np.abs(pre) ** 2).sum()
        assert abs(float(reg.sum()) - want) <= 1e-5 * want, (float(reg.sum()), want)
        ref.step({"x": (xr, torch.as_tensor(gsum) + 2 * lam * xr)})
        assert _close(tables[0].cpu().numpy(), xr.numpy(), rtol=1e-5)
    eng.close()


@pytest.mark.parametrize("W", [2, 3, 8])  # 8: the kernel's U = 2 branch; 2, 3: U = 4
@pytest.mark.parametrize("opt", list(OPTS))
def test_optimizer_step_exchange(opt, W):
    """kge_optimizer_step_exchange (phases = 0: no flag barriers) with W replicas of the [ent | rel] block and W gradient
    blocks, rank r = 0..W-1 in turn over its rows, one shard straddling the ent|rel boundary and a different regulariser
    per table (p = 2 on entities, p = 3 on relations): replicas bit-identical and bit-equal to kge_optimizer_step on the
    fp32 rank-order sum (one call per table), within 1e-5 of the legacy optimizer restatement; each rank's other gradient
    block zeroed over its whole length, the blocks read left unchanged; regulariser loss over ranks == the fp64 value."""
    from ampligraph_b200.parallel import row_shard
    from oracle import ref_step
    lib = _lib()
    name, params = OPTS[opt]
    rng = _rng(opt, W, "exchange")
    E, R, k = 97, 7, 10
    blk = E + R
    lam_e, lam_r = 1e-3, 2e-3
    eng = _engine("DistMult", k, 1, E, R, optimizer=name, optimizer_params=params,
                  regularizer=[{"p": 2, "lambda": lam_e}, {"p": 3, "lambda": lam_r}])
    ce, cr, ld = eng.opt_cfgs["ent"], eng.opt_cfgs["rel"], eng.ld
    bounds = [row_shard(blk, W, r) for r in range(W)]
    assert any(lo < E < hi for lo, hi in bounds)
    x0 = _packed(blk, ld, k, rng, 0.5)
    tables, plain = [_dev(x0) for _ in range(W)], _dev(x0)
    slots, pslots = [_opt_slots(name, params, hi - lo, ld) for lo, hi in bounds], _opt_slots(name, params, blk, ld)
    other = [torch.empty((blk, ld), device="cuda") for _ in range(W)]  # each rank's other (double-buffered) gradient block
    tp = (C.c_void_p * W)(*[x.data_ptr() for x in tables])
    cut = lambda x, lo, hi: None if x is None else x[lo:hi]
    ref, xr = ref_step.LegacyOptimizer(name, **params), torch.as_tensor(x0.copy())
    for t in (1, 2):
        gs = [_packed(blk, ld, k, rng, 1.0) for _ in range(W)]
        grads = [_dev(g) for g in gs]
        gp = (C.c_void_p * W)(*[g.data_ptr() for g in grads])
        for z in other:
            z.fill_(7.0)
        pre = tables[0].cpu().numpy().astype(np.float64)
        reg = torch.zeros(W, dtype=torch.float64, device="cuda")
        for r, (lo, hi) in enumerate(bounds):
            lib.check(eng.lib.kge_optimizer_step_exchange(
                eng.h, C.byref(ce), C.byref(cr), t, W, r, tp, gp, None, None, _ptr(other[r]), _ptr(slots[r][0]),
                _ptr(slots[r][1]), lo, hi, None, t, 0, C.c_void_p(reg.data_ptr() + 8 * r), eng._stream()))
        gsum = _rank_order_sum(gs)
        gsum_d = _dev(gsum)
        for cfg, lo, hi in ((ce, 0, E), (cr, E, blk)):
            lib.check(eng.lib.kge_optimizer_step(eng.h, C.byref(cfg), t, _ptr(plain[lo:hi]), _ptr(gsum_d[lo:hi]),
                                                 _ptr(cut(pslots[0], lo, hi)), _ptr(cut(pslots[1], lo, hi)), hi - lo, None,
                                                 eng._stream()))
        torch.cuda.synchronize()
        _check_replicas(tables, plain, slots, pslots, bounds)
        assert all((gd.cpu().numpy() == g).all() for gd, g in zip(grads, gs))
        assert all(bool((z == 0).all()) for z in other)
        want = lam_e * (np.abs(pre[:E]) ** 2).sum() + lam_r * (np.abs(pre[E:]) ** 3).sum()
        assert abs(float(reg.sum()) - want) <= 1e-5 * want, (float(reg.sum()), want)
        g_t = torch.as_tensor(gsum)
        xe, xl = xr[:E], xr[E:]
        ref.step({"ent": (xe, g_t[:E] + 2 * lam_e * xe), "rel": (xl, g_t[E:] + 3 * lam_r * xl.abs() ** 2 * torch.sign(xl))})
        assert _close(tables[0].cpu().numpy(), xr.numpy(), rtol=1e-5)
    eng.close()
