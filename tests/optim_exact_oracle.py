"""Restatement of update4 / apply_rule (ampligraph_b200/csrc/kge_optim_common.cuh) in numpy fp32, bit for bit.

Every operation is the kernel's, in the kernel's order: fma32 is a correctly rounded fp32 fma, every other +, -, * and
/ and sqrt is numpy's float32 arithmetic, which rounds to nearest as CUDA's defaults do (the library is built without
fast-math or flush-to-zero, so subnormals are kept on both sides).  1 - beta and 1 - rho are fp32 subtractions, the
bias-corrected step lr_t is formed in fp64 and rounded once (kge_api.cu, optim_params), and Adamax's max is np.fmax,
which drops a NaN as fmaxf does.  The regulariser's |x|^(p-1) is exact for p = 1, 2 and one rounding for p = 3; for
p > 3 the device's powf is not correctly rounded, so reg_grad gives the correctly rounded power and callers hold the
result to powf's documented error bound instead of equality.

Test infrastructure only: tests import it."""
from types import SimpleNamespace

import numpy as np

f32 = np.float32
KINDS = ("sgd", "adam", "adagrad", "rmsprop", "adadelta", "adamax")  # the library's KGE_OPT_* numbering
RHO_DEFAULT = {"rmsprop": 0.9, "adadelta": 0.95}


def fma32(a, b, c):
    """Correctly rounded fp32 fma(a, b, c), elementwise, IEEE semantics for signed zeros, infinities and NaN.

    The product of two fp32 values is exact in fp64 (48 significant bits, exponents well inside fp64's range).  The sum
    p + c is rounded to fp64 and its error recovered exactly with TwoSum; where the error is non-zero and the fp64 sum
    has an even last bit, the sum is moved one fp64 ulp towards the error (round to odd).  Round-to-odd at 53 bits
    followed by one rounding to 24 bits (or fewer, for a subnormal result) is the correctly rounded result.  Where p or
    c is not finite the fp64 sum is already the IEEE result, and an exact zero sum has the sign IEEE gives it."""
    a, b, c = (np.asarray(v, f32).astype(np.float64) for v in (a, b, c))
    with np.errstate(all="ignore"):
        p = a * b
        s = p + c
        bp = s - p
        e = (p - (s - bp)) + (c - bp)
        finite = np.isfinite(s) & np.isfinite(e)
        even = (s.view(np.uint64) & np.uint64(1)) == 0
        nudge = finite & (e != 0) & even
        s = np.where(nudge, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
        return s.astype(f32)


def config(name, params=None, reg=None):
    """The fields of kge_optimizer_config the rules read, with the engine's defaults (engine.KGEEngine.set_optimizer),
    each rounded to fp32 as the struct stores it.  reg: None or {"p":, "lambda": [, "p2":, "lambda2":]}."""
    p, r = dict(params or {}), dict(reg or {})
    return SimpleNamespace(
        kind=KINDS.index(name), learning_rate=f32(p.get("learning_rate", 0.001)), beta_1=f32(p.get("beta_1", 0.9)),
        beta_2=f32(p.get("beta_2", 0.999)), epsilon=f32(p.get("epsilon", 1e-7)), momentum=f32(p.get("momentum", 0.0)),
        initial_accumulator_value=f32(p.get("initial_accumulator_value", 0.1)),
        reg_p=int(r.get("p", 2)) if reg else 0, reg_lambda=f32(r.get("lambda", 1e-5)),
        reg_p2=int(r.get("p2", 0)) if reg else 0, reg_lambda2=f32(r.get("lambda2", 0.0)),
        rho=f32(p.get("rho", RHO_DEFAULT.get(name, 0.0))), centered=int(bool(p.get("centered", False))))


def lr_t(cfg, t):
    """The bias-corrected step of Adam and Adamax as kge_api.cu forms it: fp64 on the host from the fp32 fields, rounded
    to fp32 once."""
    lr, b1, b2 = float(f32(cfg.learning_rate)), float(f32(cfg.beta_1)), float(f32(cfg.beta_2))
    if KINDS[cfg.kind] == "adamax":
        return f32(lr / (1.0 - b1 ** float(t)))
    return f32(lr * np.sqrt(1.0 - b2 ** float(t)) / (1.0 - b1 ** float(t)))


def _lp_scale(ax, p, lam):
    """lam*p*|x|^(p-1) as lp_scale forms it: (lam*p)*pm1, two fp32 roundings."""
    if p == 1:
        pm1 = np.ones_like(ax)
    elif p == 2:
        pm1 = ax
    elif p == 3:
        pm1 = ax * ax
    else:
        pm1 = np.power(ax.astype(np.float64), p - 1).astype(f32)  # correctly rounded; the device's powf is not
    return (f32(lam) * f32(p)) * pm1


def reg_grad(x, p, lam, p2=0, lam2=0.0):
    """The regulariser's gradient at x (fp32): sign(x)*s1, then fma(sign(x), s2, .) for the second term; sign(+-0) and
    sign(NaN) are 0.  p = 0 (no regulariser on this table) contributes exactly +0 to nothing: returns None."""
    if p == 0:
        return None
    x = np.asarray(x, f32)
    ax = np.abs(x)
    sg = np.where(x > 0, f32(1), np.where(x < 0, f32(-1), f32(0))).astype(f32)
    with np.errstate(all="ignore"):
        g = sg * _lp_scale(ax, p, lam)
        if p2 > 0:
            g = fma32(sg, _lp_scale(ax, p2, lam2), g)
    return g


def reg_loss(x, p, lam, p2=0, lam2=0.0):
    """The exact (fp64) regulariser loss of the fp32 values x: sum of lam*|x|^p (+ lam2*|x|^p2), lam as fp32."""
    ax = np.abs(np.asarray(x, f32).astype(np.float64))
    out = float(f32(lam)) * float((ax ** p).sum()) if p else 0.0
    if p and p2:
        out += float(f32(lam2)) * float((ax ** p2).sum())
    return out


def update(cfg, t, x, g, a, b):
    """One element-wise step of cfg's rule at step t on fp32 arrays: returns new (x, a, b), the inputs unchanged.  g is the
    summed gradient the kernel reads; the regulariser's gradient (cfg.reg_p > 0) is added to it at the pre-update x.
    Slots the kind does not use come back as they went in."""
    x, g, a, b = (np.array(v, f32, copy=True) for v in (x, g, a, b))
    kind = KINDS[cfg.kind]
    lr, eps, mu, rho = f32(cfg.learning_rate), f32(cfg.epsilon), f32(cfg.momentum), f32(cfg.rho)
    one = f32(1)
    with np.errstate(all="ignore"):
        rg = reg_grad(x, cfg.reg_p, cfg.reg_lambda, cfg.reg_p2, cfg.reg_lambda2)
        if rg is not None:
            g = g + rg
        if kind == "sgd":
            if mu != 0:
                a = fma32(a, mu, -(g * lr))
                x = x + a
            else:
                x = fma32(-g, lr, x)
        elif kind == "adam":
            a = fma32(g - a, one - f32(cfg.beta_1), a)
            b = fma32(fma32(g, g, -b), one - f32(cfg.beta_2), b)
            x = x - (a * lr_t(cfg, t)) / (np.sqrt(b) + eps)
        elif kind == "adagrad":
            a = fma32(g, g, a)
            x = x - (lr * g) / (np.sqrt(a) + eps)
        elif kind == "rmsprop":
            g2, step = g * g, lr * g
            if mu != 0:
                assert not cfg.centered, "centered RMSprop with momentum is refused by the library"
                a = fma32(g2 - a, one - rho, a)
                b = fma32(mu, b, step / np.sqrt(a + eps))
                x = x - b
            else:
                a = fma32(rho, a, (one - rho) * g2)
                d = a
                if cfg.centered:
                    b = fma32(rho, b, (one - rho) * g)
                    d = fma32(-b, b, a)
                x = x - step / (np.sqrt(d) + eps)
        elif kind == "adadelta":
            a = fma32(rho, a, (one - rho) * (g * g))
            u = (np.sqrt(b + eps) / np.sqrt(a + eps)) * g
            x = fma32(-lr, u, x)
            b = fma32(rho, b, (one - rho) * (u * u))
        elif kind == "adamax":
            a = fma32(g - a, one - f32(cfg.beta_1), a)
            b = np.fmax(f32(cfg.beta_2) * b, np.abs(g))
            x = fma32(-lr_t(cfg, t), a / (b + eps), x)
        else:
            raise ValueError(kind)
    return x.astype(f32), a.astype(f32), b.astype(f32)


def uses_slots(cfg):
    """(slot 0 used, slot 1 used): the library's uses_slot0 / uses_slot1."""
    kind = KINDS[cfg.kind]
    s0 = kind != "sgd" or cfg.momentum != 0
    s1 = kind in ("adam", "adadelta", "adamax") or (kind == "rmsprop" and (bool(cfg.centered) or cfg.momentum != 0))
    return s0, s1


def bits(v):
    """fp32 values as uint32 bit patterns with every NaN made one pattern: equality of bits() is bit equality with
    NaN == NaN (the payload of a NaN is not part of the contract)."""
    u = np.asarray(v, f32).view(np.uint32).copy()
    u[np.isnan(np.asarray(v, f32))] = 0x7FC00000
    return u
