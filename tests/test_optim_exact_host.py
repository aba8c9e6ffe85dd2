"""The exact restatement of the optimizer rules (tests/optim_exact_oracle.py) on the CPU: its fma32 against exact
rational arithmetic, and the whole rules against the looser restatements of optim_oracle.rule and oracle.ref_step."""
import math
from fractions import Fraction

import numpy as np
import pytest
import torch

import optim_exact_oracle as xo
import optim_oracle
from oracle import ref_step

f32 = np.float32
FLT_MAX = float(np.finfo(f32).max)


def _round_f32(q, neg_zero):
    """The fp32 nearest to the rational q, ties to even, with IEEE overflow to inf; neg_zero: the sign of an exact 0."""
    if q == 0:
        return f32(-0.0) if neg_zero else f32(0.0)
    aq = abs(q)
    e = math.frexp(float(aq))[1] - 1  # float(aq) may be off by one binade near a power of two: fix it exactly
    while Fraction(2) ** e > aq:
        e -= 1
    while Fraction(2) ** (e + 1) <= aq:
        e += 1
    ulp = Fraction(2) ** (max(e, -126) - 23)
    v = round(aq / ulp) * ulp  # round() of a Fraction rounds half to even
    out = math.inf if v >= Fraction(2) ** 128 else float(v)
    return f32(out if q > 0 else -out)


def _fma_exact(a, b, c):
    a, b, c = (f32(v) for v in (a, b, c))
    if not (np.isfinite(a) and np.isfinite(b) and np.isfinite(c)):
        return None
    q = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    prod_neg = (np.signbit(a) != np.signbit(b))
    return _round_f32(q, neg_zero=(q == 0 and prod_neg and np.signbit(c)))


def _check(a, b, c):
    a, b, c = (np.asarray(v, f32) for v in (a, b, c))
    got = xo.fma32(a, b, c)
    for i in range(a.size):
        want = _fma_exact(a.flat[i], b.flat[i], c.flat[i])
        assert want is not None
        assert xo.bits(got.flat[i]) == xo.bits(want), (a.flat[i], b.flat[i], c.flat[i], got.flat[i], want)


def _random_f32(rng, n, emin=-140, emax=120):
    """Finite fp32 values with uniformly random significand bits and exponents in [emin, emax], random signs."""
    m = rng.integers(0, 1 << 23, n).astype(np.float64) / (1 << 23) + 1.0
    e = rng.integers(emin, emax + 1, n)
    s = rng.choice([-1.0, 1.0], n)
    return (s * np.ldexp(m, e)).astype(f32)


def test_fma32_random_triples():
    rng = np.random.default_rng(0)
    n = 4000
    a, b = _random_f32(rng, n, -70, 60), _random_f32(rng, n, -70, 60)
    c = _random_f32(rng, n, -140, 120)
    _check(a, b, c)
    # cancellation: c near -a*b, so the result keeps the product's low bits (and the residual may be tiny)
    near = (-(a.astype(np.float64) * b.astype(np.float64))).astype(f32)
    jitter = rng.integers(-3, 4, n)
    c2 = np.array([np.nextafter(v, np.inf * j) if j else v for v, j in zip(near, jitter)], f32)
    _check(a, b, c2)


def test_fma32_adversarial():
    one = 1.0 + 2.0 ** -12
    cases = [
        (one, one, 0.0),                 # exact tie 1 + 2^-11 + 2^-24: to even
        (one, one, 2.0 ** -60),          # a tie plus a tiny c: up (rounding through fp64 first would go to even)
        (one, one, -2.0 ** -60),         # ... minus a tiny c: down
        (-one, one, -2.0 ** -60),
        (1.0 + 2.0 ** -23, 1.0 + 2.0 ** -23, -1.0),  # 2^-22 + 2^-46, exact
        (2.0 ** -75, 2.0 ** -75, 0.0),   # underflows to +0
        (-2.0 ** -75, 2.0 ** -75, 0.0),  # ... keeps its sign: -0 + +0 is an exact-zero sum = +0
        (-2.0 ** -75, 2.0 ** -75, -0.0),  # -0 + -0 = -0
        (2.0 ** -75, 2.0 ** -75, 2.0 ** -149),  # subnormal c plus a product far below it
        (2.0 ** -100, 2.0 ** -49, 2.0 ** -149),  # product = 2^-149: subnormal sum 2^-148
        (2.0 ** -75, 2.0 ** -75, -2.0 ** -149),  # rounds to -2^-149, not -0
        (1.5 * 2.0 ** -75, 2.0 ** -75, 0.0),     # 1.5 * 2^-150: rounds up to 2^-149
        (2.0 ** -75, 2.0 ** -75 * 0.5, 0.0),     # 2^-151: rounds to +0
        (0.0, 5.0, -0.0), (-0.0, 5.0, -0.0), (-0.0, -5.0, -0.0), (0.0, -5.0, 0.0),
        (2.0 ** 64, 2.0 ** 64, 0.0),     # overflows to inf
        (FLT_MAX, 1.0, FLT_MAX), (FLT_MAX, -1.0, FLT_MAX), (FLT_MAX, 2.0, -FLT_MAX),
        (2.0 ** 64, 2.0 ** 64 - 2.0 ** 40, 0.0),  # 2^128 - 2^104 = FLT_MAX exactly
        (FLT_MAX, 1.0, 2.0 ** 103),      # 2^128 - 2^103: the midpoint above FLT_MAX, ties to even (odd FLT_MAX) = inf
        (FLT_MAX, 1.0, 2.0 ** 103 - 2.0 ** 79),  # just below that midpoint: FLT_MAX
        (2.0 ** 64 - 2.0 ** 40, 2.0 ** 64 - 2.0 ** 40, 0.0),
        (3.0, 1.0 / 3.0, -1.0),
    ]
    a, b, c = (np.array([x[i] for x in cases], np.float64).astype(f32) for i in range(3))
    _check(a, b, c)


@pytest.mark.parametrize("a,b,c,want", [
    (np.inf, 2.0, 1.0, np.inf), (np.inf, -2.0, 1.0, -np.inf), (np.inf, 0.0, 1.0, np.nan),
    (2.0, 3.0, np.inf, np.inf), (2.0, 3.0, -np.inf, -np.inf), (np.inf, 1.0, -np.inf, np.nan),
    (np.nan, 1.0, 1.0, np.nan), (1.0, 1.0, np.nan, np.nan), (0.0, np.nan, 0.0, np.nan),
    (FLT_MAX, FLT_MAX, -np.inf, -np.inf), (2.0 ** 100, 2.0 ** 100, -FLT_MAX, np.inf)])
def test_fma32_non_finite(a, b, c, want):
    got = xo.fma32(f32(a), f32(b), f32(c))
    assert xo.bits(got) == xo.bits(f32(want)) and np.isnan(got) == np.isnan(want)


def _ulps(got, want):
    """|got - want| in units of fp32 spacing at want, or at 1/64 of the largest |want| where want is smaller (a result
    formed by cancellation, like RMSprop's momentum, keeps the absolute error of its larger operands)."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    floor = f32(np.abs(want).max() / 64)
    sp = np.maximum(np.spacing(np.maximum(np.abs(want), floor).astype(f32)).astype(np.float64), 2.0 ** -149)
    return np.abs(got - want) / sp


NEW = [("rmsprop", {"learning_rate": 0.01}), ("rmsprop", {"learning_rate": 0.01, "rho": 0.8, "centered": True}),
       ("rmsprop", {"learning_rate": 0.01, "momentum": 0.9}), ("adadelta", {"learning_rate": 1.0}),
       ("adamax", {"learning_rate": 0.01})]
OLD = [("sgd", {"learning_rate": 0.01}), ("sgd", {"learning_rate": 0.01, "momentum": 0.9}),
       ("adam", {"learning_rate": 0.01}), ("adagrad", {"learning_rate": 0.01})]


@pytest.mark.parametrize("name,params", NEW + OLD)
def test_restatement_vs_oracles(name, params):
    """Three steps on ordinary U(-1, 1) inputs: the exact restatement and optim_oracle.rule / ref_step.LegacyOptimizer
    agree within a few ulp of the result.  They are not bit-equal: ref_step forms SGD, Adam and Adagrad in another order
    (and Adam's betas in fp64), and both run on torch's CPU sqrt, which is not correctly rounded (numpy's is)."""
    rng = np.random.default_rng(len(name) * 7 + len(params))
    n = 2000
    cfg = xo.config(name, params)
    x = rng.uniform(-1, 1, n).astype(f32)
    a = np.full(n, cfg.initial_accumulator_value if name == "adagrad" else 0.0, f32)
    b = np.zeros(n, f32)
    xt, at, bt = (torch.from_numpy(v.copy()) for v in (x, a, b))
    opt = ref_step.LegacyOptimizer(name, params["learning_rate"], **{k: v for k, v in params.items() if k != "learning_rate"})
    for t in (1, 2, 3):
        g = rng.uniform(-1, 1, n).astype(f32)
        x, a, b = xo.update(cfg, t, x, g, a, b)
        if name in optim_oracle.NEW_KINDS:
            optim_oracle.rule(name, xt, torch.from_numpy(g), at, bt, t, params["learning_rate"], params)
        else:
            opt.t = t
            opt.apply(xt, torch.from_numpy(g), "x")
    assert _ulps(x, xt.numpy()).max() <= 32, _ulps(x, xt.numpy()).max()
    if name in optim_oracle.NEW_KINDS:
        s0, s1 = xo.uses_slots(cfg)
        assert not s0 or _ulps(a, at.numpy()).max() <= 32
        assert not s1 or _ulps(b, bt.numpy()).max() <= 32


def test_restatement_regulariser():
    """reg_grad for p in {1, 2, 3} and the pair (1, 2) on ordinary values and at +-0 equals the fp64 derivative rounded
    the kernel's way; at +-0 the p = 1 gradient is exactly +0 (sign(0) = 0), and the update sees g + reg."""
    rng = np.random.default_rng(5)
    x = np.concatenate([rng.uniform(-2, 2, 500), [0.0, -0.0]]).astype(f32)
    lam = f32(1e-3)
    for p in (1, 2, 3):
        got = xo.reg_grad(x, p, lam)
        want = float(lam) * p * np.abs(x.astype(np.float64)) ** (p - 1) * np.sign(x)
        assert _ulps(got, want).max() <= 3
        assert (xo.bits(got[-2:]) == 0).all()  # +0 at both zeros
    g12 = xo.reg_grad(x, 1, lam, 2, f32(2e-3))
    want = float(lam) * np.sign(x) + 2 * 2e-3 * x.astype(np.float64)
    assert _ulps(g12, want).max() <= 4
    cfg = xo.config("sgd", {"learning_rate": 0.5}, {"p": 1, "lambda": 1e-3})
    xn, _, _ = xo.update(cfg, 1, x, np.zeros_like(x), x, x)
    assert (xo.bits(xn) == xo.bits(xo.fma32(-(xo.reg_grad(x, 1, lam)), f32(0.5), x))).all()
    assert xo.reg_grad(x, 0, lam) is None


def test_lr_t_matches_host_formula():
    cfg = xo.config("adam", {"learning_rate": 0.01, "beta_1": 0.8, "beta_2": 0.99})
    lr, b1, b2 = (float(f32(v)) for v in (0.01, 0.8, 0.99))  # the config's fp32 fields, widened on the host
    for t in (1, 2, 1000, 10 ** 6):
        want = np.float32(lr * math.sqrt(1 - b2 ** t) / (1 - b1 ** t))
        assert abs(float(xo.lr_t(cfg, t)) - float(want)) <= float(np.spacing(want)) * 1.01
