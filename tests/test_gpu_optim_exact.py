"""The optimizer rules on the GPU, element by element and bit for bit, against tests/optim_exact_oracle.py.

Every optimizer path inlines the one update4 of kge_optim_common.cuh, so path-against-path equality cannot see a wrong
rule: here each path is compared with the fp32 restatement, with no tolerance (NaN equals NaN), on inputs drawn from
the rules' edges -- signed zeros, subnormals, values whose square underflows or overflows, values near sqrt(eps),
FLT_MAX, infinities and NaN -- with pad columns that must stay +0 and gradients that must come back zeroed.  The
regulariser's loss, an fp32 sum per thread and per warp, is held to a derived bound."""
import ctypes as C
import itertools
import zlib

import numpy as np
import pytest
import torch

import optim_exact_oracle as xo
from ampligraph_b200 import _lib

pytestmark = pytest.mark.gpu

f32 = np.float32
FLT_MAX = float(np.finfo(f32).max)
# x, g and first-moment slots: any value
POOL = np.array([0.0, -0.0, 2.0 ** -149, -2.0 ** -149, 1e-40, -3e-39, 1e-23, -3e-22, 3.1622776e-4, -3.2e-4, 1e-5,
                 0.5, -1.25, 3.0, 1e20, -3e19, FLT_MAX, -FLT_MAX, np.inf, -np.inf, np.nan], f32)
# second-moment slots: their valid domain, >= 0
POS = np.array([0.0, 2.0 ** -149, 1e-40, 1e-20, 1e-10, 1e-7, 0.25, 3.0, 1e30, FLT_MAX, np.inf], f32)

CASES = {
    "sgd": ("sgd", {"learning_rate": 0.01}),
    "sgd_momentum": ("sgd", {"learning_rate": 0.01, "momentum": 0.9}),
    "adam": ("adam", {}),
    "adam_eps1e-10": ("adam", {"learning_rate": 0.01, "epsilon": 1e-10}),
    "adam_eps1": ("adam", {"epsilon": 1.0, "beta_1": 0.5, "beta_2": 0.9}),
    "adagrad": ("adagrad", {"learning_rate": 0.01}),
    "adagrad_eps1e-10": ("adagrad", {"learning_rate": 0.01, "epsilon": 1e-10}),
    "rmsprop": ("rmsprop", {}),
    "rmsprop_centered": ("rmsprop", {"learning_rate": 0.01, "rho": 0.8, "centered": True}),
    "rmsprop_momentum": ("rmsprop", {"learning_rate": 0.01, "momentum": 0.5, "epsilon": 1e-10}),
    "adadelta": ("adadelta", {"learning_rate": 1.0}),
    "adadelta_rho": ("adadelta", {"learning_rate": 0.5, "rho": 0.5, "epsilon": 1.0}),
    "adamax": ("adamax", {}),
    "adamax_b2": ("adamax", {"learning_rate": 0.01, "beta_2": 0.5, "epsilon": 1e-10}),
}
REGS = [None, {"p": 1, "lambda": 1e-3}, {"p": 2, "lambda": 1e-2}, {"p": 3, "lambda": 1e-3},
        {"p": 1, "lambda": 1e-3, "p2": 2, "lambda2": 2e-3}]
K, LD = 13, 16  # DistMult k = 13: rows of stride 16, three pad columns


def _engine(*a, **kw):
    from ampligraph_b200.engine import KGEEngine
    return KGEEngine(*a, **kw)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a)).cuda().contiguous()


def _second_moments(cfg):
    """(slot 0 is a second moment, slot 1 is one): their draws come from POS."""
    kind = xo.KINDS[cfg.kind]
    s0 = kind in ("adagrad", "rmsprop", "adadelta")
    s1 = kind in ("adam", "adadelta", "adamax")
    return s0, s1


def _edge_inputs(cfg, rows, seed):
    """[rows, LD] fp32 x, g, slot 0, slot 1 with +0 pads: a Cartesian block of (x, g, slot) picks first, then random
    picks from the pools."""
    rng = np.random.default_rng(seed)
    m0, m1 = _second_moments(cfg)
    n = rows * K
    x, g = rng.choice(POOL, n), rng.choice(POOL, n)
    s0, s1 = rng.choice(POS if m0 else POOL, n), rng.choice(POS if m1 else POOL, n)
    cart = np.array(list(itertools.product(POOL, POOL, POS if (m0 or m1) else POOL)), f32)
    c = min(len(cart), n)
    x[:c], g[:c] = cart[:c, 0], cart[:c, 1]
    if m0 or not m1:
        s0[:c] = cart[:c, 2]
    if m1:
        s1[:c] = cart[:c, 2]

    def pack(v):
        out = np.zeros((rows, LD), f32)
        out[:, :K] = v.reshape(rows, K)
        return out
    return pack(x), pack(g), pack(s0), pack(s1)


def _cfg(eng, key="ent"):
    return eng.opt_cfgs[key]


def _expect(cfg, t, x, g, a, b):
    """The restatement over whole [rows, LD] arrays; slots the kind does not use stay as given."""
    u0, u1 = xo.uses_slots(cfg)
    nx, na, nb = xo.update(cfg, t, x, g, a, b)
    return nx, (na if u0 else a), (nb if u1 else b)


def _assert_bits(got, want, what):
    got = got.detach().cpu().numpy() if torch.is_tensor(got) else got
    bad = xo.bits(got) != xo.bits(want)
    if bad.any():
        i = np.argwhere(bad)[0]
        raise AssertionError("%s: %d elements differ, first at %s: got %r want %r" %
                             (what, int(bad.sum()), tuple(i), got[tuple(i)], want[tuple(i)]))


def _make(name, params, reg, E=4080, R=16, eta=1):
    eng = _engine("DistMult", K, eta, E, R, optimizer=name, optimizer_params=params, regularizer=reg)
    assert eng.ld == LD
    return eng


def _slots_of(cfg, a, b):
    u0, u1 = xo.uses_slots(cfg)
    return (_dev(a) if u0 else None), (_dev(b) if u1 else None)


CASE_IDS = list(CASES)


@pytest.mark.parametrize("t", [1, 2, 1000, 10 ** 6])
@pytest.mark.parametrize("case", CASE_IDS)
def test_dense_edges(case, t):
    name, params = CASES[case]
    eng = _make(name, params, None)
    rows = eng.n_ent + eng.n_rel
    cfg = _cfg(eng)
    x, g, a, b = _edge_inputs(cfg, rows, zlib.crc32(repr((case, t)).encode()))
    dx, dg = _dev(x), _dev(g)
    d0, d1 = _slots_of(cfg, a, b)
    _lib.check(eng.lib.kge_optimizer_step(eng.h, C.byref(cfg), t, _ptr(dx), _ptr(dg), _ptr(d0), _ptr(d1), rows, None,
                                          eng._stream()))
    torch.cuda.synchronize()
    wx, wa, wb = _expect(cfg, t, x, g, a, b)
    _assert_bits(dx, wx, "x")
    if d0 is not None:
        _assert_bits(d0, wa, "slot 0")
    if d1 is not None:
        _assert_bits(d1, wb, "slot 1")
    _assert_bits(dg, np.zeros_like(g), "gradient zeroed")
    assert (xo.bits(dx.cpu().numpy()[:, K:]) == 0).all()  # pads stay +0
    eng.close()


@pytest.mark.parametrize("reg", REGS[1:], ids=lambda r: "p%d_%d" % (r["p"], r.get("p2", 0)))
@pytest.mark.parametrize("case", ["sgd", "sgd_momentum", "adam", "adagrad", "rmsprop_centered", "adadelta", "adamax"])
def test_dense_edges_regularised(case, reg):
    """The regulariser's gradient at the pre-update x, added to g: exact for p in {1, 2, 3} and the pair (1, 2), at
    +-0 (sign 0), at infinities and NaN."""
    name, params = CASES[case]
    eng = _make(name, params, reg)
    rows = eng.n_ent + eng.n_rel
    cfg = _cfg(eng)
    assert cfg.reg_p == reg["p"]
    x, g, a, b = _edge_inputs(cfg, rows, zlib.crc32(repr((case, str(reg))).encode()))
    dx, dg = _dev(x), _dev(g)
    d0, d1 = _slots_of(cfg, a, b)
    loss = torch.zeros(1, dtype=torch.float64, device="cuda")
    _lib.check(eng.lib.kge_optimizer_step(eng.h, C.byref(cfg), 3, _ptr(dx), _ptr(dg), _ptr(d0), _ptr(d1), rows,
                                          _ptr(loss), eng._stream()))
    torch.cuda.synchronize()
    wx, wa, wb = _expect(cfg, 3, x, g, a, b)
    _assert_bits(dx, wx, "x")
    if d0 is not None:
        _assert_bits(d0, wa, "slot 0")
    if d1 is not None:
        _assert_bits(d1, wb, "slot 1")
    _assert_bits(dg, np.zeros_like(g), "gradient zeroed")
    eng.close()


def test_dense_regulariser_p4_within_powf_bound():
    """p = 4: the device's powf is not correctly rounded; the CUDA C++ Programming Guide's table of single-precision
    functions bounds powf's error by 4 ulp.  The restatement's |x|^3 is correctly rounded (0.5 ulp), so the two differ by
    at most 4.5 ulp of |x|^3.  Both multiply it by the same fp32 c = lam*p and round once (the products differ by at most
    c * 4.5 ulp of |x|^3, plus one ulp of the product where the rounding goes different ways), and then form
    x - s with one rounding (lr = 1), which adds at most one ulp of the result."""
    eng = _make("sgd", {"learning_rate": 1.0}, {"p": 4, "lambda": 0.1})
    rows = eng.n_ent + eng.n_rel
    cfg = _cfg(eng)
    rng = np.random.default_rng(4)
    x = np.zeros((rows, LD), f32)
    x[:, :K] = rng.uniform(-2, 2, (rows, K))
    dx, dg = _dev(x), _dev(np.zeros_like(x))
    _lib.check(eng.lib.kge_optimizer_step(eng.h, C.byref(cfg), 1, _ptr(dx), _ptr(dg), None, None, rows, None,
                                          eng._stream()))
    torch.cuda.synchronize()
    want, _, _ = xo.update(cfg, 1, x, np.zeros_like(x), x, x)
    c = float(f32(cfg.reg_lambda) * f32(4))
    pm1 = np.abs(x.astype(np.float64)) ** 3
    s_ = c * pm1
    bound = (c * 4.5 * np.spacing(pm1.astype(f32)).astype(np.float64) + np.spacing(s_.astype(f32)).astype(np.float64)
             + np.spacing(np.abs(want)).astype(np.float64))
    assert (np.abs(dx.cpu().numpy().astype(np.float64) - want) <= bound).all()
    eng.close()


@pytest.mark.parametrize("t", [1, 10 ** 6])
@pytest.mark.parametrize("case", ["sgd", "sgd_momentum", "adam_eps1e-10", "adagrad", "rmsprop_momentum",
                                  "rmsprop_centered", "adadelta", "adamax"])
def test_lazy_edges(case, t):
    """Stamped rows take the rule; unstamped rows, their slots and their gradients stay bit-unchanged."""
    name, params = CASES[case]
    eng = _make(name, params, None)
    rows = eng.n_ent + eng.n_rel
    cfg = _cfg(eng)
    x, g, a, b = _edge_inputs(cfg, rows, zlib.crc32(repr(("lazy", case, t)).encode()))
    stamped = np.random.default_rng(t).random(rows) < 0.5
    stamp = 7
    stamps = _dev(np.where(stamped, stamp, stamp - 1).astype(np.int32))
    dx, dg = _dev(x), _dev(g)
    d0, d1 = _slots_of(cfg, a, b)
    _lib.check(eng.lib.kge_optimizer_step_lazy(eng.h, C.byref(cfg), t, _ptr(dx), _ptr(dg), _ptr(d0), _ptr(d1), rows,
                                               _ptr(stamps), stamp, None, eng._stream()))
    torch.cuda.synchronize()
    wx, wa, wb = _expect(cfg, t, x, g, a, b)
    sel = lambda new, old: np.where(stamped[:, None], new, old)
    _assert_bits(dx, sel(wx, x), "x")
    if d0 is not None:
        _assert_bits(d0, sel(wa, a), "slot 0")
    if d1 is not None:
        _assert_bits(d1, sel(wb, b), "slot 1")
    _assert_bits(dg, sel(np.zeros_like(g), g), "gradient")
    eng.close()


@pytest.mark.parametrize("W", [1, 3])
@pytest.mark.parametrize("case", ["sgd", "adam", "adagrad_eps1e-10", "rmsprop_centered", "adadelta_rho", "adamax_b2"])
def test_sharded_edges(case, W):
    """kge_optimizer_step_sharded with the gradient on rank 0 and +0 on the others: the rank-order sum starts from +0,
    so the rule sees (+0 + g) -- a -0 gradient becomes +0 -- and every replica gets the same rows."""
    from ampligraph_b200.parallel import row_shard
    name, params = CASES[case]
    eng = _make(name, params, {"p": 2, "lambda": 1e-2})
    rows = eng.n_ent + eng.n_rel
    cfg = _cfg(eng)
    x, g, a, b = _edge_inputs(cfg, rows, zlib.crc32(repr(("sharded", case, W)).encode()))
    tables = [_dev(x) for _ in range(W)]
    grads = [_dev(g)] + [torch.zeros_like(tables[0]) for _ in range(W - 1)]
    tp = (C.c_void_p * W)(*[v.data_ptr() for v in tables])
    gp = (C.c_void_p * W)(*[v.data_ptr() for v in grads])
    u0, u1 = xo.uses_slots(cfg)
    shards = []
    for r in range(W):
        lo, hi = row_shard(rows, W, r)
        s0 = _dev(a[lo:hi]) if u0 and hi > lo else None
        s1 = _dev(b[lo:hi]) if u1 and hi > lo else None
        shards.append((lo, hi, s0, s1))
        _lib.check(eng.lib.kge_optimizer_step_sharded(eng.h, C.byref(cfg), 5, W, r, tp, gp, _ptr(s0), _ptr(s1), lo, hi,
                                                      None, eng._stream()))
    torch.cuda.synchronize()
    wx, wa, wb = _expect(cfg, 5, x, f32(0) + g, a, b)
    for v in tables:
        _assert_bits(v, wx, "replica")
    for lo, hi, s0, s1 in shards:
        if s0 is not None:
            _assert_bits(s0, wa[lo:hi], "slot 0 shard")
        if s1 is not None:
            _assert_bits(s1, wb[lo:hi], "slot 1 shard")
    eng.close()


def _exchange(eng, ce, cr, t, W, x, g, a, b, loss=None):
    """kge_optimizer_step_exchange (phases 0) for ranks 0..W-1 in turn; the gradient on rank 0, +0 elsewhere."""
    from ampligraph_b200.parallel import row_shard
    rows = eng.n_ent + eng.n_rel
    tables = [_dev(x) for _ in range(W)]
    grads = [_dev(g)] + [torch.zeros_like(tables[0]) for _ in range(W - 1)]
    tp = (C.c_void_p * W)(*[v.data_ptr() for v in tables])
    gp = (C.c_void_p * W)(*[v.data_ptr() for v in grads])
    u0, u1 = xo.uses_slots(ce)
    shards = []
    for r in range(W):
        lo, hi = row_shard(rows, W, r)
        s0 = _dev(a[lo:hi]) if u0 and hi > lo else None
        s1 = _dev(b[lo:hi]) if u1 and hi > lo else None
        shards.append((lo, hi, s0, s1))
        _lib.check(eng.lib.kge_optimizer_step_exchange(eng.h, C.byref(ce), C.byref(cr), t, W, r, tp, gp, None, None, None,
                                                       _ptr(s0), _ptr(s1), lo, hi, None, t, 0,
                                                       None if loss is None else _ptr(loss),
                                                       eng._stream()))
    torch.cuda.synchronize()
    return tables, shards


EXCHANGE_REGS = {"p2_p12": [{"p": 2, "lambda": 1e-2}, {"p": 1, "lambda": 1e-3, "p2": 2, "lambda2": 2e-3}],
                 "p3_p1": [{"p": 3, "lambda": 1e-3}, {"p": 1, "lambda": 1e-3}]}


@pytest.mark.parametrize("regs", list(EXCHANGE_REGS))
@pytest.mark.parametrize("W", [1, 3, 8])  # 8: the kernel's U = 2 branch
@pytest.mark.parametrize("case", ["sgd_momentum", "adam", "adagrad", "rmsprop", "rmsprop_momentum", "adadelta", "adamax"])
def test_exchange_edges(case, W, regs):
    """phases 0, a different regulariser per table (entities p = 2 or 3, relations the pair (1, 2) or p = 1); at W = 1
    the rule sees g itself, at W > 1 the rank-order sum g + (+0)."""
    name, params = CASES[case]
    E = 4080
    eng = _make(name, params, EXCHANGE_REGS[regs])
    ce, cr = _cfg(eng, "ent"), _cfg(eng, "rel")
    rows = eng.n_ent + eng.n_rel
    x, g, a, b = _edge_inputs(ce, rows, zlib.crc32(repr(("exchange", case, W, regs)).encode()))
    tables, shards = _exchange(eng, ce, cr, 9, W, x, g, a, b)
    gs = g if W == 1 else g + f32(0)
    we = _expect(ce, 9, x[:E], gs[:E], a[:E], b[:E])
    wr = _expect(cr, 9, x[E:], gs[E:], a[E:], b[E:])
    wx, wa, wb = (np.concatenate([p, q]) for p, q in zip(we, wr))
    for v in tables:
        _assert_bits(v, wx, "replica")
    for lo, hi, s0, s1 in shards:
        if s0 is not None:
            _assert_bits(s0, wa[lo:hi], "slot 0 shard")
        if s1 is not None:
            _assert_bits(s1, wb[lo:hi], "slot 1 shard")
    eng.close()


def test_exchange_unregularised_table():
    """A table without a regulariser next to one with it (the reference's LP on the entities only): its rows take the
    plain rule -- its zeros and pads stay finite -- and it adds nothing to the regulariser loss."""
    E = 4080
    eng = _make("adam", {"learning_rate": 0.01}, [{"p": 2, "lambda": 1e-2}, None])
    ce, cr = _cfg(eng, "ent"), _cfg(eng, "rel")
    assert ce.reg_p == 2 and cr.reg_p == 0
    rows = eng.n_ent + eng.n_rel
    rng = np.random.default_rng(2)
    x = np.zeros((rows, LD), f32)
    x[:, :K] = rng.uniform(-1, 1, (rows, K))
    x[E:, :3] = 0.0
    g = np.zeros_like(x)
    g[:, :K] = rng.uniform(-1, 1, (rows, K))
    a, b = np.zeros_like(x), np.zeros_like(x)
    loss = torch.zeros(1, dtype=torch.float64, device="cuda")
    tables, _ = _exchange(eng, ce, cr, 1, 1, x, g, a, b, loss)
    we = _expect(ce, 1, x[:E], g[:E], a[:E], b[:E])
    wr = _expect(cr, 1, x[E:], g[E:], a[E:], b[E:])
    _assert_bits(tables[0], np.concatenate([we[0], wr[0]]), "x")
    _check_loss(float(loss.item()), [(x[:E, :K], 2, ce.reg_lambda, 0, 0.0)], rows * LD // 4)
    eng.close()


def _check_loss(got, terms, n4):
    """The regulariser loss against its fp64 value.  Each element's term lam*|x|^p (+ lam2*|x|^p2) is formed with at most
    3 fp32 roundings (|x|*|x|, *|x|, and lam in the fma that adds it), so it is within gamma_3 of its exact value.  A
    thread adds its terms into one fp32 sum with the fma; a thread of a kernel of any grid takes at most ceil(n4/256)
    float4s, i.e. 4*2*ceil(n4/256) terms, then 5 levels of warp shuffles add fp32 partial sums: every term passes
    through at most D = 8*ceil(n4/256) + 5 fp32 additions, so the fp32 part is within gamma_D of the sum of the
    (positive) rounded terms (Higham, Accuracy and Stability, 4.2).  The block sums and the atomics are fp64: within
    gamma_{n4} in fp64.  Subnormal terms add at most 2^-149 each absolutely."""
    u, u64 = 2.0 ** -24, 2.0 ** -53
    S = sum(xo.reg_loss(v, p, lam, p2, lam2) for v, p, lam, p2, lam2 in terms)
    n = sum(v.size for v, *_ in terms)
    D = 8 * -(-n4 // 256) + 5
    gam = lambda m, uu=u: m * uu / (1 - m * uu)
    bound = (gam(3) + gam(D) * (1 + gam(3))) * S * (1 + gam(n4, u64)) + 3 * n * 2.0 ** -149
    assert abs(got - S) <= bound, (got, S, bound)


@pytest.mark.parametrize("regs", [({"p": 1, "lambda": 1e-3}, {"p": 3, "lambda": 2e-3}),
                                  ({"p": 2, "lambda": 1e-2}, {"p": 1, "lambda": 1e-3, "p2": 2, "lambda2": 2e-3})])
def test_regulariser_loss_within_bound(regs):
    """The dense kernel (one table) and the exchange kernel (a different regulariser per table) on ordinary values."""
    E = 4080
    eng = _make("sgd", {"learning_rate": 0.01}, list(regs))
    ce, cr = _cfg(eng, "ent"), _cfg(eng, "rel")
    rows = eng.n_ent + eng.n_rel
    rng = np.random.default_rng(8)
    x = np.zeros((rows, LD), f32)
    x[:, :K] = rng.uniform(-1, 1, (rows, K))
    g = np.zeros_like(x)
    z = np.zeros_like(x)
    loss = torch.zeros(1, dtype=torch.float64, device="cuda")
    dx, dg = _dev(x), _dev(g)
    _lib.check(eng.lib.kge_optimizer_step(eng.h, C.byref(ce), 1, _ptr(dx), _ptr(dg), None, None, rows, _ptr(loss),
                                          eng._stream()))
    torch.cuda.synchronize()
    r = regs[0]
    _check_loss(float(loss.item()), [(x[:, :K], r["p"], ce.reg_lambda, r.get("p2", 0), ce.reg_lambda2)], rows * LD // 4)
    loss.zero_()
    _exchange(eng, ce, cr, 1, 1, x, g, z, z, loss)
    re_, rr = regs
    _check_loss(float(loss.item()), [(x[:E, :K], re_["p"], ce.reg_lambda, re_.get("p2", 0), ce.reg_lambda2),
                                     (x[E:, :K], rr["p"], cr.reg_lambda, rr.get("p2", 0), cr.reg_lambda2)],
                rows * LD // 4)
    eng.close()


@pytest.mark.parametrize("t,reg", [(1, None), (1000, None), (7, {"p": 3, "lambda": 1e-3}),
                                   (7, {"p": 1, "lambda": 1e-3, "p2": 2, "lambda2": 2e-3})],
                         ids=["t1", "t1000", "t7_p3", "t7_p12"])
@pytest.mark.parametrize("case", ["sgd", "sgd_momentum", "adam", "adagrad", "rmsprop_centered", "rmsprop_momentum",
                                  "adadelta", "adamax"])
def test_deferred_owner_edges(case, t, reg):
    """The owner-per-row kernel of a deferred DistMult step, with and without a regulariser.  The step's positives and
    corruptions use only all-zero carrier rows (entities 0..3, relation 0), so every term it forms is +-0 and the edge
    rows have empty buckets; their gradients are written into the gradient block before kge_optimizer_step_deferred,
    whose rule sees g + (+0)."""
    name, params = CASES[case]
    E, R, B, eta = 4080, 16, 1024, 4
    eng = _make(name, params, reg, E, R, eta)
    cfg = _cfg(eng)
    rows = E + R
    x, g, a, b = _edge_inputs(cfg, rows, zlib.crc32(repr(("deferred", case, t, str(reg))).encode()))
    carrier = np.zeros(rows, bool)
    carrier[:4] = carrier[E] = True
    x[carrier] = 0.0
    rng = np.random.default_rng(t)
    trip = np.stack([rng.integers(0, 4, B), np.zeros(B, np.int64), rng.integers(0, 4, B)], 1).astype(np.int32)
    neg = (_dev(rng.integers(0, 4, B * eta).astype(np.int32)), _dev(rng.integers(0, 2, B * eta).astype(np.uint8)))
    eng._pblock.copy_(_dev(x))
    u0, u1 = xo.uses_slots(cfg)
    if u0:
        eng._sblocks[0].copy_(_dev(a))
    if u1:
        eng._sblocks[1].copy_(_dev(b))
    eng.forward_backward(_dev(trip), neg, step=0, defer=True)
    assert eng._deferred
    edge = torch.as_tensor(~carrier).cuda()
    eng._gblock[edge] = _dev(g)[edge]
    eng.t = t - 1
    eng.apply_gradients()
    torch.cuda.synchronize()
    assert eng.t == t
    wx, wa, wb = _expect(cfg, t, x, g + f32(0), a, b)
    keep = ~carrier
    _assert_bits(eng._pblock.cpu().numpy()[keep], wx[keep], "x")
    if u0:
        _assert_bits(eng._sblocks[0].cpu().numpy()[keep], wa[keep], "slot 0")
    if u1:
        _assert_bits(eng._sblocks[1].cpu().numpy()[keep], wb[keep], "slot 1")
    _assert_bits(eng._gblock.cpu().numpy(), np.zeros_like(g), "gradient zeroed")
    eng.close()


def test_centered_rmsprop_constant_gradient():
    """~200 steps of centered RMSprop with a constant gradient: mg^2 approaches ms, and d = ms - mg^2 can round below 0,
    where sqrt gives NaN (Keras legacy forms the same d).  The kernel follows the restatement step for step, NaN
    included; the test records whether NaN appears without asserting either way."""
    eng = _make("rmsprop", {"learning_rate": 0.01, "centered": True}, None)
    cfg = _cfg(eng)
    rows = eng.n_ent + eng.n_rel
    rng = np.random.default_rng(200)
    x = np.zeros((rows, LD), f32)
    x[:, :K] = rng.uniform(-1, 1, (rows, K))
    g = np.zeros_like(x)
    g[:, :K] = rng.choice(np.array([1.0, -0.3, 1e-3, 7.5, 1e-20, 3e15], f32), (rows, K))
    a, b = np.zeros_like(x), np.zeros_like(x)
    dx, d0, d1 = _dev(x), _dev(a), _dev(b)
    dg_const = _dev(g)
    for t in range(1, 201):
        dg = dg_const.clone()
        _lib.check(eng.lib.kge_optimizer_step(eng.h, C.byref(cfg), t, _ptr(dx), _ptr(dg), _ptr(d0), _ptr(d1), rows, None,
                                              eng._stream()))
        x, a, b = xo.update(cfg, t, x, g, a, b)
    torch.cuda.synchronize()
    _assert_bits(dx, x, "x")
    _assert_bits(d0, a, "ms")
    _assert_bits(d1, b, "mg")
    print("centered RMSprop, 200 constant-gradient steps: %d of %d elements NaN" % (int(np.isnan(x).sum()), x.size))
    eng.close()


# ---------------------------------------------------------------------------
# whole steps through the engine
# ---------------------------------------------------------------------------
STEP_CASES = dict(CASES, adagrad_iav0=("adagrad", {"learning_rate": 0.01, "initial_accumulator_value": 0.0}))
STEP_REG = {"p": 2, "lambda": 2.0 ** -10}


@pytest.mark.parametrize("path", ["dense", "deferred", "lazy"])
@pytest.mark.parametrize("case,reg", [(c, None) for c in ("sgd", "sgd_momentum", "adam", "adagrad", "adagrad_iav0",
                                                            "rmsprop", "rmsprop_centered", "rmsprop_momentum", "adadelta",
                                                            "adamax")]
                         + [(c, STEP_REG) for c in ("adam", "rmsprop_centered", "adamax")],
                         ids=lambda v: v if isinstance(v, str) else ("reg" if v else "noreg"))
def test_engine_steps_exact(case, reg, path):
    """Three engine steps (DistMult, pairwise loss) on exact_oracle's dyadic tables, where every gradient sum is exact in
    any order, so the gradients the optimizer reads equal the float64 oracle's.  The tables are reset to fresh dyadic
    tables before each step (an update leaves the grid); the slots, initialised by the engine, and its t carry over.
    After each step the tables and slots equal the restatement applied to the oracle's gradients with the engine's t:
    dense (bucket sum, then kge_optimizer_step), deferred (the owner-per-row kernel) and lazy (looked-up rows only)."""
    import exact_oracle as eo
    from ampligraph_b200.engine import optimizer_slots
    name, params = STEP_CASES[case]
    rng = np.random.default_rng(zlib.crc32(repr((case, str(reg), path)).encode()))
    k, E, R, B, eta = 33, 500, 9, 1000, 4
    lp = {"margin": 1.0, "reduction": "sum"}
    eng = _engine("DistMult", k, eta, E, R, loss="pairwise", loss_params=lp,
                  optimizer=("lazy_" if path == "lazy" else "") + name, optimizer_params=params, regularizer=reg)
    assert eng.ld > k  # pad columns exist
    init = optimizer_slots(eng.opt_cfg)
    state = {key: [np.full((n, k), 0.0 if v is None else v, f32) for v in init] for key, n in (("ent", E), ("rel", R))}
    u0, u1 = xo.uses_slots(eng.opt_cfg)
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
        ref = eo.oracle_step("DistMult", ent, rel, t, eta, ne, nk, loss="pairwise", loss_params=lp)
        touched = {"ent": np.unique(np.concatenate([t[:, 0], t[:, 2], ne])), "rel": np.unique(t[:, 1])}
        got = dict(zip(("ent", "rel"), eng.get_embeddings()))
        for key, x0, gref in (("ent", ent, ref.g_ent), ("rel", rel, ref.g_rel)):
            eo.assert_fp32_exact(gref, "oracle gradient")
            g = gref.numpy().astype(f32) + f32(0)
            a, b = state[key]
            nx, na, nb = xo.update(eng.opt_cfgs[key], eng.t, x0, g, a, b)
            if path == "lazy":
                rows = np.zeros(len(x0), bool)
                rows[touched[key]] = True
                keep = lambda new, old: np.where(rows[:, None], new, old)
                nx, na, nb = keep(nx, x0), keep(na, a), keep(nb, b)
            state[key] = [na if u0 else a, nb if u1 else b]
            _assert_bits(got[key], nx, "%s table, step %d" % (key, step))
            for j, used in enumerate((u0, u1)):
                if used:
                    _assert_bits(eng.slots[key][j][:, :k], state[key][j], "%s slot %d, step %d" % (key, j, step))
        assert (xo.bits(eng._pblock.cpu().numpy()[:, k:]) == 0).all()  # pads stay +0
    eng.close()
