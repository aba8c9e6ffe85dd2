"""Nadam and Ftrl on the GPU, element by element and bit for bit against tests/nadam_ftrl_oracle.py, on every path the
two kinds reach: dense, Nadam's row-decay mode, lazy, regularised tables, sharded and exchange steps, the deferred
owner-per-row kernel and whole engine steps; at the rules' edges (signed zeros, subnormals, FLT_MAX, infinities, NaN),
Nadam's looked-up row with a zero gradient and untouched row with m != 0, Ftrl's |z| == l1, the pow path, ApplyFtrlV2's
shrinkage and beta > 0.  Then the config layouts and refusals, a fit with each optimizer, and save / load."""
import ctypes as C
import itertools
import zlib

import numpy as np
import pytest
import torch

import nadam_ftrl_oracle as nfo
import optim_exact_oracle as xo
from ampligraph_b200 import _lib

pytestmark = pytest.mark.gpu

f32 = np.float32
FLT_MAX = float(np.finfo(f32).max)
POOL = np.array([0.0, -0.0, 2.0 ** -149, -2.0 ** -149, 1e-40, -3e-39, 1e-23, -3e-22, 3.1622776e-4, -3.2e-4, 1e-5,
                 0.5, -1.25, 3.0, 1e20, -3e19, FLT_MAX, -FLT_MAX, np.inf, -np.inf, np.nan], f32)
POS = np.array([0.0, 2.0 ** -149, 1e-40, 1e-20, 1e-10, 1e-7, 0.25, 3.0, 1e30, FLT_MAX, np.inf], f32)
CASES = {
    "nadam": ("nadam", {}),
    "nadam_b": ("nadam", {"learning_rate": 0.01, "beta_1": 0.5, "beta_2": 0.9, "epsilon": 1e-10, "decay": 0.1}),
    "ftrl": ("ftrl", {"learning_rate": 0.05}),
    "ftrl_l1": ("ftrl", {"learning_rate": 0.05, "l1_regularization_strength": 0.5}),
    "ftrl_pow": ("ftrl", {"learning_rate": 0.05, "learning_rate_power": -0.25, "l1_regularization_strength": 1e-3}),
    "ftrl_pow15": ("ftrl", {"learning_rate": 0.5, "learning_rate_power": -1.5}),
    "ftrl_v2": ("ftrl", {"learning_rate": 0.05, "l2_shrinkage_regularization_strength": 0.1,
                         "l2_regularization_strength": 0.01}),
    "ftrl_beta": ("ftrl", {"learning_rate": 0.05, "beta": 0.5, "l2_regularization_strength": 0.01,
                           "initial_accumulator_value": 0.0}),
}
REGS = [{"p": 1, "lambda": 1e-3}, {"p": 2, "lambda": 1e-2}, {"p": 3, "lambda": 1e-3},
        {"p": 1, "lambda": 1e-3, "p2": 2, "lambda2": 2e-3}]
K, LD = 13, 16  # DistMult k = 13: rows of stride 16, three pad columns


def _engine(*a, **kw):
    from ampligraph_b200.engine import KGEEngine
    return KGEEngine(*a, **kw)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a)).cuda().contiguous()


def _pow_dev(y, e):
    """powf on the device (torch's fp32 pow is CUDA's powf), the power the kernel's pow path takes."""
    y = _dev(np.asarray(y, f32))
    return torch.pow(y, torch.full_like(y, float(e))).cpu().numpy()


def _expect(cfg, t, x, g, a, b, moved=None):
    return nfo.update(cfg, t, x, g, a, b, moved=moved, pow32=_pow_dev)


def _edge_inputs(cfg, rows, seed):
    """[rows, LD] x, g, slot 0, slot 1 with +0 pads: a Cartesian block of picks, then random picks.  The second-moment
    slot (Nadam's v, Ftrl's n) draws from POS."""
    rng = np.random.default_rng(seed)
    nadam = nfo.KINDS[cfg.kind] == "nadam"
    n = rows * K
    x, g = rng.choice(POOL, n), rng.choice(POOL, n)
    s0, s1 = rng.choice(POOL if nadam else POS, n), rng.choice(POS if nadam else POOL, n)
    cart = np.array(list(itertools.product(POOL, POOL, POS)), f32)
    c = min(len(cart), n)
    x[:c], g[:c] = cart[:c, 0], cart[:c, 1]
    (s1 if nadam else s0)[:c] = cart[:c, 2]

    def pack(v):
        out = np.zeros((rows, LD), f32)
        out[:, :K] = v.reshape(rows, K)
        return out
    return pack(x), pack(g), pack(s0), pack(s1)


def _assert_bits(got, want, what):
    got = got.detach().cpu().numpy() if torch.is_tensor(got) else got
    bad = xo.bits(got) != xo.bits(want)
    if bad.any():
        i = np.argwhere(bad)[0]
        raise AssertionError("%s: %d elements differ, first at %s: got %r want %r" %
                             (what, int(bad.sum()), tuple(i), got[tuple(i)], want[tuple(i)]))


def _make(case, reg=None, E=4080, R=16, eta=1, t=1, cache=0.75, **kw):
    """An engine for the case whose configs hold step t's scalars (Nadam: from momentum cache `cache`)."""
    name, params = CASES[case]
    eng = _engine("DistMult", K, eta, E, R, optimizer=name, optimizer_params=params, regularizer=reg, **kw)
    assert eng.ld == LD
    eng.t, eng.nadam_cache = t - 1, f32(cache)
    eng.begin_step()
    assert eng.t == t
    return eng


CASE_IDS = list(CASES)


@pytest.mark.parametrize("t", [1, 2, 1000, 10 ** 6])
@pytest.mark.parametrize("case", CASE_IDS)
def test_dense_edges(case, t):
    eng = _make(case, t=t)
    cfg = eng.opt_cfg
    rows = eng.n_ent + eng.n_rel
    x, g, a, b = _edge_inputs(cfg, rows, zlib.crc32(repr((case, t)).encode()))
    dx, dg, d0, d1 = _dev(x), _dev(g), _dev(a), _dev(b)
    _lib.check(eng.lib.kge_optimizer_step(eng.h, C.byref(cfg), t, _ptr(dx), _ptr(dg), _ptr(d0), _ptr(d1), rows, None,
                                          eng._stream()))
    torch.cuda.synchronize()
    wx, wa, wb = _expect(cfg, t, x, g, a, b)
    _assert_bits(dx, wx, "x")
    _assert_bits(d0, wa, "slot 0")
    _assert_bits(d1, wb, "slot 1")
    _assert_bits(dg, np.zeros_like(g), "gradient zeroed")
    assert (xo.bits(dx.cpu().numpy()[:, K:]) == 0).all()  # pads stay +0
    eng.close()


@pytest.mark.parametrize("reg", REGS, ids=lambda r: "p%d_%d" % (r["p"], r.get("p2", 0)))
@pytest.mark.parametrize("case", ["nadam", "ftrl_l1", "ftrl_v2", "ftrl_pow"])
def test_dense_edges_regularised(case, reg):
    eng = _make(case, reg, t=3)
    cfg = eng.opt_cfg
    assert cfg.reg_p == reg["p"]
    rows = eng.n_ent + eng.n_rel
    x, g, a, b = _edge_inputs(cfg, rows, zlib.crc32(repr((case, str(reg))).encode()))
    dx, dg, d0, d1 = _dev(x), _dev(g), _dev(a), _dev(b)
    loss = torch.zeros(1, dtype=torch.float64, device="cuda")
    _lib.check(eng.lib.kge_optimizer_step(eng.h, C.byref(cfg), 3, _ptr(dx), _ptr(dg), _ptr(d0), _ptr(d1), rows,
                                          _ptr(loss), eng._stream()))
    torch.cuda.synchronize()
    wx, wa, wb = _expect(cfg, 3, x, g, a, b)
    _assert_bits(dx, wx, "x")
    _assert_bits(d0, wa, "slot 0")
    _assert_bits(d1, wb, "slot 1")
    _assert_bits(dg, np.zeros_like(g), "gradient zeroed")
    eng.close()


@pytest.mark.parametrize("t", [1, 7, 10 ** 6])
@pytest.mark.parametrize("case", ["nadam", "nadam_b"])
def test_nadam_decay_mode_edges(case, t):
    """kge_optimizer_step_decay: stamped rows take the dense rule, unstamped rows only decay m and v; their table and
    gradient rows are not written.  A stamped row with an exactly zero gradient moves; an unstamped row with m != 0
    does not."""
    eng = _make(case, t=t)
    cfg = eng.opt_cfg
    rows = eng.n_ent + eng.n_rel
    x, g, a, b = _edge_inputs(cfg, rows, zlib.crc32(repr(("decay", case, t)).encode()))
    stamped = np.random.default_rng(t).random(rows) < 0.5
    stamped[:2] = [True, False]
    g[0, :K], a[0, :K], b[0, :K], x[0, :K] = 0.0, 0.5, 0.25, 1.0  # looked up, zero gradient, m != 0
    a[1, :K], b[1, :K], x[1, :K] = -0.5, 0.25, 1.0  # not looked up, m != 0
    g[~stamped] = 0.0  # the stamping contract: a row that was not looked up has no gradient
    g[1, :3] = 7.0  # ... but were it there, the decay mode would neither read nor clear it
    stamp = 11
    stamps = _dev(np.where(stamped, stamp, stamp + 1).astype(np.int32))
    dx, dg, d0, d1 = _dev(x), _dev(g), _dev(a), _dev(b)
    _lib.check(eng.lib.kge_optimizer_step_decay(eng.h, C.byref(cfg), t, _ptr(dx), _ptr(dg), _ptr(d0), _ptr(d1), rows,
                                                _ptr(stamps), stamp, eng._stream()))
    torch.cuda.synchronize()
    wx, wa, wb = _expect(cfg, t, x, g, a, b, moved=stamped[:, None])
    _assert_bits(dx, wx, "x")
    _assert_bits(d0, wa, "m")
    _assert_bits(d1, wb, "v")
    _assert_bits(dg, np.where(stamped[:, None], f32(0), g), "gradient")
    got = dx.cpu().numpy()
    assert (got[0, :K] != 1.0).all() and (got[1, :K] == 1.0).all()
    eng.close()


@pytest.mark.parametrize("t", [1, 10 ** 6])
@pytest.mark.parametrize("case", CASE_IDS)
def test_lazy_edges(case, t):
    """lazy_nadam / lazy_ftrl: stamped rows take the rule; unstamped rows, their slots and gradients stay unchanged."""
    eng = _make(case, t=t)
    cfg = eng.opt_cfg
    rows = eng.n_ent + eng.n_rel
    x, g, a, b = _edge_inputs(cfg, rows, zlib.crc32(repr(("lazy", case, t)).encode()))
    stamped = np.random.default_rng(t).random(rows) < 0.5
    stamp = 7
    stamps = _dev(np.where(stamped, stamp, stamp - 1).astype(np.int32))
    dx, dg, d0, d1 = _dev(x), _dev(g), _dev(a), _dev(b)
    _lib.check(eng.lib.kge_optimizer_step_lazy(eng.h, C.byref(cfg), t, _ptr(dx), _ptr(dg), _ptr(d0), _ptr(d1), rows,
                                               _ptr(stamps), stamp, None, eng._stream()))
    torch.cuda.synchronize()
    wx, wa, wb = _expect(cfg, t, x, g, a, b)
    sel = lambda new, old: np.where(stamped[:, None], new, old)
    _assert_bits(dx, sel(wx, x), "x")
    _assert_bits(d0, sel(wa, a), "slot 0")
    _assert_bits(d1, sel(wb, b), "slot 1")
    _assert_bits(dg, sel(np.zeros_like(g), g), "gradient")
    eng.close()


@pytest.mark.parametrize("W", [1, 3])
@pytest.mark.parametrize("case", ["nadam_b", "ftrl_l1", "ftrl_pow", "ftrl_v2"])
def test_sharded_edges(case, W):
    """kge_optimizer_step_sharded (one GPU, W simulated ranks): gradient on rank 0, +0 elsewhere; every replica gets
    the restatement's rows."""
    from ampligraph_b200.parallel import row_shard
    eng = _make(case, {"p": 2, "lambda": 1e-2}, t=5)
    cfg = eng.opt_cfg
    rows = eng.n_ent + eng.n_rel
    x, g, a, b = _edge_inputs(cfg, rows, zlib.crc32(repr(("sharded", case, W)).encode()))
    tables = [_dev(x) for _ in range(W)]
    grads = [_dev(g)] + [torch.zeros_like(tables[0]) for _ in range(W - 1)]
    tp = (C.c_void_p * W)(*[v.data_ptr() for v in tables])
    gp = (C.c_void_p * W)(*[v.data_ptr() for v in grads])
    shards = []
    for r in range(W):
        lo, hi = row_shard(rows, W, r)
        s0, s1 = _dev(a[lo:hi]), _dev(b[lo:hi])
        shards.append((lo, hi, s0, s1))
        _lib.check(eng.lib.kge_optimizer_step_sharded(eng.h, C.byref(cfg), 5, W, r, tp, gp, _ptr(s0), _ptr(s1), lo, hi,
                                                      None, eng._stream()))
    torch.cuda.synchronize()
    wx, wa, wb = _expect(cfg, 5, x, f32(0) + g, a, b)
    for v in tables:
        _assert_bits(v, wx, "replica")
    for lo, hi, s0, s1 in shards:
        _assert_bits(s0, wa[lo:hi], "slot 0 shard")
        _assert_bits(s1, wb[lo:hi], "slot 1 shard")
    eng.close()


@pytest.mark.parametrize("W", [1, 3])
@pytest.mark.parametrize("case", ["nadam", "ftrl_l1", "ftrl_pow15", "ftrl_beta"])
def test_exchange_edges(case, W):
    """kge_optimizer_step_exchange, phases 0, a regulariser on the entities only."""
    from ampligraph_b200.parallel import row_shard
    E = 4080
    eng = _make(case, [{"p": 2, "lambda": 1e-2}, None], t=9)
    ce, cr = eng.opt_cfgs["ent"], eng.opt_cfgs["rel"]
    rows = eng.n_ent + eng.n_rel
    x, g, a, b = _edge_inputs(ce, rows, zlib.crc32(repr(("exchange", case, W)).encode()))
    tables = [_dev(x) for _ in range(W)]
    grads = [_dev(g)] + [torch.zeros_like(tables[0]) for _ in range(W - 1)]
    tp = (C.c_void_p * W)(*[v.data_ptr() for v in tables])
    gp = (C.c_void_p * W)(*[v.data_ptr() for v in grads])
    shards = []
    for r in range(W):
        lo, hi = row_shard(rows, W, r)
        s0, s1 = _dev(a[lo:hi]), _dev(b[lo:hi])
        shards.append((lo, hi, s0, s1))
        _lib.check(eng.lib.kge_optimizer_step_exchange(eng.h, C.byref(ce), C.byref(cr), 9, W, r, tp, gp, None, None, None,
                                                       _ptr(s0), _ptr(s1), lo, hi, None, 9, 0, None, eng._stream()))
    torch.cuda.synchronize()
    gs = g if W == 1 else g + f32(0)
    we = _expect(ce, 9, x[:E], gs[:E], a[:E], b[:E])
    wr = _expect(cr, 9, x[E:], gs[E:], a[E:], b[E:])
    wx, wa, wb = (np.concatenate([p, q]) for p, q in zip(we, wr))
    for v in tables:
        _assert_bits(v, wx, "replica")
    for lo, hi, s0, s1 in shards:
        _assert_bits(s0, wa[lo:hi], "slot 0 shard")
        _assert_bits(s1, wb[lo:hi], "slot 1 shard")
    eng.close()


@pytest.mark.parametrize("t,reg", [(1, None), (1000, None), (7, {"p": 3, "lambda": 1e-3})], ids=["t1", "t1000", "t7_p3"])
@pytest.mark.parametrize("case", ["nadam", "ftrl", "ftrl_pow", "ftrl_v2"])
def test_deferred_owner_edges(case, t, reg):
    """The owner-per-row kernel of a deferred DistMult step instantiates both kinds: the step's rows are all-zero
    carrier rows (every term it forms is +-0), the edge rows' gradients are written before apply_gradients, whose rule
    sees g + (+0) with the engine's own step scalars."""
    name, params = CASES[case]
    E, R, B, eta = 4080, 16, 1024, 4
    eng = _engine("DistMult", K, eta, E, R, optimizer=name, optimizer_params=params, regularizer=reg)
    assert eng.table_rules == {"ent": "dense", "rel": "dense"}
    rows = E + R
    x, g, a, b = _edge_inputs(eng.opt_cfg, rows, zlib.crc32(repr(("deferred", case, t, str(reg))).encode()))
    carrier = np.zeros(rows, bool)
    carrier[:4] = carrier[E] = True
    x[carrier] = 0.0
    rng = np.random.default_rng(t)
    trip = np.stack([rng.integers(0, 4, B), np.zeros(B, np.int64), rng.integers(0, 4, B)], 1).astype(np.int32)
    neg = (_dev(rng.integers(0, 4, B * eta).astype(np.int32)), _dev(rng.integers(0, 2, B * eta).astype(np.uint8)))
    eng._pblock.copy_(_dev(x))
    eng._sblocks[0].copy_(_dev(a))
    eng._sblocks[1].copy_(_dev(b))
    eng.forward_backward(_dev(trip), neg, step=0, defer=True)
    assert eng._deferred
    edge = torch.as_tensor(~carrier).cuda()
    eng._gblock[edge] = _dev(g)[edge]
    eng.t, eng.nadam_cache = t - 1, f32(0.6)
    eng.apply_gradients()
    torch.cuda.synchronize()
    assert eng.t == t
    wx, wa, wb = _expect(eng.opt_cfg, t, x, g + f32(0), a, b)
    keep = ~carrier
    _assert_bits(eng._pblock.cpu().numpy()[keep], wx[keep], "x")
    _assert_bits(eng._sblocks[0].cpu().numpy()[keep], wa[keep], "slot 0")
    _assert_bits(eng._sblocks[1].cpu().numpy()[keep], wb[keep], "slot 1")
    _assert_bits(eng._gblock.cpu().numpy(), np.zeros_like(g), "gradient zeroed")
    eng.close()


def test_ftrl_l1_boundary_and_untouched_rows():
    """|z| == l1 exactly leaves x at 0, one ulp above moves it; a row without a gradient at step 1 (z = 0) becomes 0."""
    eng = _make("ftrl_l1")
    cfg = eng.opt_cfg
    rows = eng.n_ent + eng.n_rel
    x = np.zeros((rows, LD), f32)
    x[:, :K] = 0.7
    g = np.zeros_like(x)
    n = np.zeros_like(x)
    n[:, :K] = 0.1
    z = np.zeros_like(x)
    z[0, :4] = [0.5, -0.5, np.nextafter(f32(0.5), f32(1)), np.nextafter(f32(-0.5), f32(-1))]
    x[0, :4] = 0.0  # z moves by -sigma * x = 0: the new z is the given one
    dx, dg, d0, d1 = _dev(x), _dev(g), _dev(n), _dev(z)
    _lib.check(eng.lib.kge_optimizer_step(eng.h, C.byref(cfg), 1, _ptr(dx), _ptr(dg), _ptr(d0), _ptr(d1), rows, None,
                                          eng._stream()))
    torch.cuda.synchronize()
    got = dx.cpu().numpy()
    _assert_bits(got, _expect(cfg, 1, x, g, n, z)[0], "x")
    assert got[0, 0] == 0 and got[0, 1] == 0 and got[0, 2] < 0 < got[0, 3]
    assert (xo.bits(got[1:]) == 0).all()  # untouched rows with z = 0: +0
    eng.close()


# ---------------------------------------------------------------------------
# whole steps through the engine
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("path", ["dense", "deferred", "decay", "lazy"])
@pytest.mark.parametrize("case,reg", [("nadam", None), ("nadam_b", None), ("ftrl", None), ("ftrl_pow", None),
                                      ("ftrl_v2", None), ("nadam", {"p": 2, "lambda": 2.0 ** -10}),
                                      ("ftrl_beta", {"p": 2, "lambda": 2.0 ** -10})],
                         ids=lambda v: v if isinstance(v, str) else ("reg" if v else "noreg"))
def test_engine_steps_exact(case, reg, path):
    """Three engine steps (DistMult, pairwise loss) on exact_oracle's dyadic tables, where every gradient sum is exact,
    so the optimizer reads the float64 oracle's gradients.  Tables reset before each step; the slots, t and Nadam's cache
    carry over, and the step's scalars come from the engine (begin_step, once per step for both tables).  dense, deferred
    (owner-per-row kernel), decay (Nadam's IndexedSlices rule, kge_optimizer_step_decay) and lazy."""
    import exact_oracle as eo
    from ampligraph_b200.engine import nadam_coefficients, optimizer_slots
    name, params = CASES[case]
    if path == "decay" and (name != "nadam" or reg):
        pytest.skip("the row-decay rule is Nadam's, on a table without a regulariser")
    rng = np.random.default_rng(zlib.crc32(repr((case, str(reg), path)).encode()))
    k, E, R, B, eta = 33, 500, 9, 1000, 4
    lp = {"margin": 1.0, "reduction": "sum"}
    eng = _engine("DistMult", k, eta, E, R, loss="pairwise", loss_params=lp,
                  optimizer=("lazy_" if path == "lazy" else "") + name, optimizer_params=params, regularizer=reg,
                  lazy_tables=(True, True) if path == "decay" else None)
    want_rule = {"dense": "dense", "deferred": "dense", "decay": "decay", "lazy": "rows"}[path]
    assert eng.table_rules == {"ent": want_rule, "rel": want_rule}
    init = optimizer_slots(eng.opt_cfg)
    state = {key: [np.full((n, k), v, f32) for v in init] for key, n in (("ent", E), ("rel", R))}
    cache = f32(1.0)
    for step in range(3):
        ent, rel = eo.grid_table(rng, E, k), eo.grid_table(rng, R, k)
        eng.set_embeddings(ent, rel)
        t = eo.zipf_triples(E, R, B, rng)
        ne = rng.integers(0, E, B * eta).astype(np.int32)
        nk = rng.integers(0, 2, B * eta).astype(np.uint8)
        eng.forward_backward(_dev(t), (_dev(ne), _dev(nk)), step=step, defer=path == "deferred")
        assert eng._deferred == (path == "deferred")
        eng.apply_gradients()
        torch.cuda.synchronize()
        assert eng.t == step + 1
        if name == "nadam":
            co = nadam_coefficients(eng.opt_cfg.beta_1, eng.opt_cfg.beta_2, eng.nadam_decay, eng.t, cache)
            cache = co[2]
            assert eng.nadam_cache == cache
            for cfg in eng.opt_cfgs.values():
                assert (cfg.nadam_m_t, cfg.nadam_m_t1, cfg.nadam_s_new, cfg.nadam_s_next, cfg.nadam_v_den) == co
        ref = eo.oracle_step("DistMult", ent, rel, t, eta, ne, nk, loss="pairwise", loss_params=lp)
        touched = {"ent": np.unique(np.concatenate([t[:, 0], t[:, 2], ne])), "rel": np.unique(t[:, 1])}
        got = dict(zip(("ent", "rel"), eng.get_embeddings()))
        for key, x0, gref in (("ent", ent, ref.g_ent), ("rel", rel, ref.g_rel)):
            eo.assert_fp32_exact(gref, "oracle gradient")
            g = gref.numpy().astype(f32) + f32(0)
            a, b = state[key]
            rows = np.zeros(len(x0), bool)
            rows[touched[key]] = True
            if path == "decay":
                nx, na, nb = _expect(eng.opt_cfgs[key], eng.t, x0, g, a, b, moved=rows[:, None])
            else:
                nx, na, nb = _expect(eng.opt_cfgs[key], eng.t, x0, g, a, b)
            if path == "lazy":
                keep = lambda new, old: np.where(rows[:, None], new, old)
                nx, na, nb = keep(nx, x0), keep(na, a), keep(nb, b)
            state[key] = [na, nb]
            _assert_bits(got[key], nx, "%s table, step %d" % (key, step))
            for j in range(2):
                _assert_bits(eng.slots[key][j][:, :k], state[key][j], "%s slot %d, step %d" % (key, j, step))
        assert (xo.bits(eng._pblock.cpu().numpy()[:, k:]) == 0).all()  # pads stay +0
    eng.close()


# ---------------------------------------------------------------------------
# layouts, refusals, the facade
# ---------------------------------------------------------------------------
def _prefix_config(cfg, stop):
    """A copy of cfg in the older layout that ends before field `stop` (struct_size = its offset)."""
    fields = []
    for f, ty in _lib.KgeOptimizerConfig._fields_:
        if f == stop:
            break
        fields.append((f, ty))
    Old = type("Old_" + stop, (C.Structure,), {"_fields_": fields})
    old = Old(*[getattr(cfg, f) for f, _ in fields])
    old.struct_size = C.sizeof(Old)
    return old


@pytest.mark.parametrize("stop,kinds", [("rho", ("sgd", "adam", "adagrad")),
                                        ("l1", ("adam", "rmsprop", "adadelta", "adamax"))])
def test_older_config_layouts(stop, kinds):
    """Both older layouts drive the kinds they knew bit-identically to the current one; Nadam or Ftrl in either is
    refused and launches nothing."""
    rng = np.random.default_rng(5)
    rows = 64
    for name in kinds + ("nadam", "ftrl"):
        eng = _engine("DistMult", K, 1, rows - 4, 4, optimizer=name, optimizer_params={"learning_rate": 0.01})
        cfg = eng.opt_cfg
        eng.begin_step()
        old = _prefix_config(cfg, stop)
        assert old.struct_size == {"rho": 48, "l1": 56}[stop]
        x = np.zeros((rows, LD), f32)
        x[:, :K] = rng.uniform(-1, 1, (rows, K))
        g = np.zeros_like(x)
        g[:, :K] = rng.uniform(-1, 1, (rows, K))
        runs = []
        for c in (cfg, old):
            dx, dg = _dev(x), _dev(g)
            s = [_dev(np.full_like(x, 0.1)), _dev(np.zeros_like(x))]
            call = lambda: _lib.check(eng.lib.kge_optimizer_step(
                eng.h, C.cast(C.pointer(c), C.POINTER(_lib.KgeOptimizerConfig)), 1, _ptr(dx), _ptr(dg), _ptr(s[0]),
                _ptr(s[1]), rows, None, eng._stream()))
            if c is old and name in ("nadam", "ftrl"):
                with pytest.raises(ValueError, match="optimizer identifier"):
                    call()
                torch.cuda.synchronize()
                _assert_bits(dx, x, "refused: table untouched")
                _assert_bits(dg, g, "refused: gradient untouched")
                continue
            call()
            torch.cuda.synchronize()
            runs.append([v.cpu().numpy() for v in (dx, s[0], s[1])])
        if len(runs) == 2:
            for p_, q_ in zip(*runs):
                _assert_bits(q_, p_, "%s in the layout before %s" % (name, stop))
        eng.close()


def test_refusals():
    """kge_optimizer_step_decay is Nadam's and refuses a regularised table; Ftrl's hyper-parameters are checked by the
    engine and the library; the replicated trainer refuses Nadam's IndexedSlices rule like the lazy rules."""
    from ampligraph_b200.parallel import reject_lazy
    rows = 32
    eng = _engine("DistMult", K, 1, rows - 4, 4, optimizer="adam")
    z = _dev(np.zeros((rows, LD), f32))
    st = _dev(np.zeros(rows, np.int32))
    decay = lambda cfg: _lib.check(eng.lib.kge_optimizer_step_decay(eng.h, C.byref(cfg), 1, _ptr(z), _ptr(z), _ptr(z),
                                                                   _ptr(z), rows, _ptr(st), 1, eng._stream()))
    with pytest.raises(NotImplementedError):
        decay(eng.opt_cfg)
    eng.set_optimizer("nadam", regularizer={"p": 2, "lambda": 1e-3})
    with pytest.raises(ValueError):
        decay(eng.opt_cfg)
    eng.set_optimizer("ftrl")
    cfg = eng.opt_cfg
    cfg.lr_power = 0.5
    with pytest.raises(ValueError):
        _lib.check(eng.lib.kge_optimizer_step(eng.h, C.byref(cfg), 1, _ptr(z), _ptr(z), _ptr(z), _ptr(z), rows, None,
                                              eng._stream()))
    for bad in ({"learning_rate_power": 0.5}, {"l1_regularization_strength": -1.0},
                {"l2_shrinkage_regularization_strength": -0.1}, {"initial_accumulator_value": -1.0}):
        with pytest.raises(ValueError):
            eng.set_optimizer("ftrl", bad)
    eng.set_optimizer("nadam", lazy_tables=(False, True))
    assert eng.table_rules == {"ent": "dense", "rel": "decay"} and eng.lazy
    with pytest.raises(NotImplementedError):
        reject_lazy("lazy_" if eng.lazy else "", 2)
    eng.set_optimizer("lazy_nadam")
    assert eng.table_rules == {"ent": "rows", "rel": "rows"}
    # a config switched to another kind behind set_optimizer's back: refused before the step starts
    eng.opt_cfgs["rel"].kind = _lib.OPTIMIZERS["ftrl"]
    with pytest.raises(ValueError, match="set_optimizer"):
        eng.apply_gradients()
    assert eng.t == 0
    eng.close()


def _kg(E, R, n, seed=1):
    rng = np.random.default_rng(seed)
    t = np.unique(np.stack([rng.integers(0, E, n), rng.integers(0, R, n), rng.integers(0, E, n)], 1), axis=0)
    rng.shuffle(t)
    return np.stack([np.char.add("e", t[:, 0].astype(str)), np.char.add("r", t[:, 1].astype(str)),
                     np.char.add("e", t[:, 2].astype(str))], 1)


def _model(optimizer, params, reg_ent):
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel, loss_functions, optimizers, regularizers
    m = ScoringBasedEmbeddingModel(eta=3, k=16, scoring_type="ComplEx", seed=7)
    m.compile(optimizer=optimizers.OptimizerWrapper(optimizer, dict(params)), loss=loss_functions.get("nll"),
              entity_relation_regularizer=[regularizers.LP_regularizer({"p": 2, "lambda": 1e-4}) if reg_ent else None,
                                           None])
    return m


@pytest.mark.parametrize("optimizer,params,reg_ent,rules", [
    ("nadam", {"learning_rate": 0.01}, False, {"ent": "decay", "rel": "decay"}),
    ("nadam", {"learning_rate": 0.01}, True, {"ent": "dense", "rel": "decay"}),
    ("ftrl", {"learning_rate": 0.5}, False, {"ent": "dense", "rel": "dense"}),
    ("ftrl", {"learning_rate": 0.5, "l1_regularization_strength": 1e-4, "beta": 0.1}, True,
     {"ent": "dense", "rel": "dense"})])
def test_fit_lowers_loss_and_save_load_resumes(optimizer, params, reg_ent, rules, tmp_path):
    """fit on a small graph lowers the loss with the reference's per-table rules; then save_weights / load_weights and
    two more optimizer steps equal the run that kept going, bit for bit (both apply the same fixed gradients, so the
    comparison sees exactly the restored tables, slots, t and Nadam's momentum cache)."""
    from ampligraph_b200.datasets import DataIndexer
    X = _kg(200, 12, 2000, seed=3)
    m = _model(optimizer, params, reg_ent)
    hist = m.fit(X, batch_size=500, epochs=6, verbose=False)
    losses = hist.history["loss"]
    assert losses[-1] < losses[0], losses
    assert m.engine.table_rules == rules

    def fixed_steps(eng, first):
        rng = np.random.default_rng(first)
        for step in range(first, first + 2):
            eng._gblock.copy_(_dev(rng.uniform(-1, 1, tuple(eng._gblock.shape)).astype(f32)))  # ComplEx k = 16: no pads
            stamp = eng.lib.kge_step_stamp(step)
            for key in ("ent", "rel"):
                if eng.stamps[key] is not None:
                    eng.stamps[key].copy_(_dev(np.where(rng.random(eng.stamps[key].numel()) < 0.5, stamp, 0)
                                               .astype(np.int32)))
            eng._last_step = step
            eng.apply_gradients()
        torch.cuda.synchronize()

    fixed_steps(m.engine, 100)
    path = str(tmp_path / "w.pkl")
    m.save_weights(path)
    fixed_steps(m.engine, 102)
    m2 = _model(optimizer, params, reg_ent)
    m2.load_weights(path)
    assert m2.engine.t == m.engine.t - 2 and m2.engine.table_rules == rules
    fixed_steps(m2.engine, 102)
    assert m2.engine.t == m.engine.t and m2.engine.nadam_cache == m.engine.nadam_cache
    for a, b in zip(m2.engine.get_embeddings(), m.engine.get_embeddings()):
        _assert_bits(a, b.cpu().numpy(), "table after load + 2 steps")
    for key in ("ent", "rel"):
        for a, b in zip(m2.engine.slots[key], m.engine.slots[key]):
            _assert_bits(a, b.cpu().numpy(), "%s slot after load + 2 steps" % key)
    if optimizer == "nadam":
        assert m.engine.nadam_cache != 1.0
