"""Restatement of the Nadam and Ftrl branches of apply_rule (ampligraph_b200/csrc/kge_optim_common.cuh) in numpy fp32, bit
for bit, and of the per-step scalars they read: Nadam's (engine.nadam_coefficients) and Ftrl's adjusted l2 (kge_api.cu,
optim_step).

Both rules round every operation on its own; numpy's float32 +, -, *, / and sqrt round to nearest as CUDA's defaults do.
Ftrl's power P(y) = y^(-lr_power) for lr_power != -0.5 is the device's powf, which is not correctly rounded: callers
pass the power function to use (the GPU tests pass one that evaluates powf on the device); the default is the correctly
rounded power.  Nadam's row-decay mode (kge_optimizer_step_decay) is `moved`: a row that was not looked up only decays m
and v.  The other six kinds are optim_exact_oracle's.

Test infrastructure only: tests import it."""
from fractions import Fraction

import numpy as np

import optim_exact_oracle as xo

f32 = np.float32
KINDS = xo.KINDS + ("nadam", "ftrl")  # the library's KGE_OPT_* numbering


def pow_rn(y, e):
    """fp32 y ** e, elementwise, correctly rounded up to an fp64 double rounding."""
    with np.errstate(all="ignore"):
        return np.power(np.asarray(y, f32).astype(np.float64), float(f32(e))).astype(f32)


def ftrl_l2x2(cfg):
    """2 * (l2 + beta / (2 lr)), every operation in fp32 (Keras' adjusted l2, then ApplyFtrl's 2 * l2)."""
    two = f32(2)
    return two * (f32(cfg.l2) + f32(cfg.ftrl_beta) / (two * f32(cfg.learning_rate)))


def update(cfg, t, x, g, a, b, moved=None, pow32=pow_rn):
    """One element-wise step of cfg's rule at step t on fp32 arrays -> new (x, a, b); the inputs are unchanged.  g is
    the summed gradient the kernel reads; the regulariser's gradient (cfg.reg_p > 0) is added at the pre-update x.
    moved: None (every row moves) or a bool array broadcastable to x: Nadam's row-decay mode, where the False rows only
    decay m and v.  Nadam reads the step's scalars from cfg (nadam_*); t is used by the other kinds only."""
    kind = KINDS[cfg.kind]
    if kind not in ("nadam", "ftrl"):
        assert moved is None
        return xo.update(cfg, t, x, g, a, b)
    x, g, a, b = (np.array(v, f32, copy=True) for v in (x, g, a, b))
    one, lr = f32(1), f32(cfg.learning_rate)
    with np.errstate(all="ignore"):
        rg = xo.reg_grad(x, cfg.reg_p, cfg.reg_lambda, cfg.reg_p2, cfg.reg_lambda2)
        if rg is not None:
            g = g + rg
        if kind == "nadam":
            b1, b2, eps = f32(cfg.beta_1), f32(cfg.beta_2), f32(cfg.epsilon)
            na = b1 * a + (one - b1) * g
            nb = b2 * b + (one - b2) * (g * g)
            mb = (one - f32(cfg.nadam_m_t)) * (g / (one - f32(cfg.nadam_s_new))) + \
                f32(cfg.nadam_m_t1) * (na / (one - f32(cfg.nadam_s_next)))
            nx = x - (lr * mb) / (np.sqrt(nb / f32(cfg.nadam_v_den)) + eps)
            if moved is not None:
                mv = np.broadcast_to(np.asarray(moved, bool), x.shape)
                nx = np.where(mv, nx, x)
                na = np.where(mv, na, b1 * a)
                nb = np.where(mv, nb, b2 * b)
            return nx.astype(f32), na.astype(f32), nb.astype(f32)
        assert moved is None
        p = f32(cfg.lr_power)
        shrinkx2 = f32(2) * f32(cfg.l2_shrinkage)
        gs = g + shrinkx2 * x if shrinkx2 > 0 else g
        n1 = a + g * g
        P = np.sqrt if p == f32(-0.5) else (lambda y: pow32(y, -p))
        p1, p0 = P(n1), P(a)
        z = b + (gs - ((p1 - p0) / lr) * x)
        den = p1 / lr + ftrl_l2x2(cfg)
        l1 = f32(cfg.l1)
        nx = np.where(np.abs(z) > l1, (np.copysign(l1, z) - z) / den, f32(0))
        return nx.astype(f32), n1.astype(f32), z.astype(f32)


def uses_slots(cfg):
    """(slot 0 used, slot 1 used): the library's uses_slot0 / uses_slot1."""
    if KINDS[cfg.kind] in ("nadam", "ftrl"):
        return True, True
    return xo.uses_slots(cfg)


def _round32(q):
    """The fp32 value nearest to the rational q (ties to even), subnormals included, for |q| below fp32's overflow."""
    if q == 0:
        return f32(0)
    sgn, a = (-1 if q < 0 else 1), abs(q)
    e = 0
    while a >= 2:
        a /= 2
        e += 1
    while a < 1:
        a *= 2
        e -= 1
    quantum = Fraction(2) ** (max(e, -126) - 23)  # the spacing of fp32 values at |q|
    m = abs(q) / quantum
    n = int(m)
    r = m - n
    if r > Fraction(1, 2) or (r == Fraction(1, 2) and n % 2 == 1):
        n += 1
    return f32(sgn * float(n * quantum))


def _pow_exact(base, e):
    """base ** e for fp32 base and exponent, correctly rounded to fp32 through 60-digit arithmetic."""
    import mpmath
    with mpmath.workdps(60):
        v = mpmath.power(mpmath.mpf(float(base)), mpmath.mpf(float(e)))
        man, exp = int(v.man), int(v.exp)  # v = man * 2^exp exactly
        return _round32(Fraction(man) * Fraction(2) ** exp)


def nadam_coefficients_exact(beta_1, beta_2, decay, t, cache):
    """engine.nadam_coefficients restated with exact rational fp32 arithmetic (every +, -, * rounded once to fp32 from its
    exact value) and a correctly rounded pow: (m_t, m_t1, s_new, s_next, v_den)."""
    F = lambda v: Fraction(float(v))
    r = lambda q: _round32(q)
    b1, d, c = f32(beta_1), f32(decay), f32(cache)

    def m(step):
        e = r(F(d) * F(f32(step)))
        return r(F(b1) * F(r(1 - F(r(F(0.5) * F(_pow_exact(f32(0.96), e)))))))
    m_t, m_t1 = m(t), m(t + 1)
    s_new = r(F(c) * F(m_t))
    return m_t, m_t1, s_new, r(F(s_new) * F(m_t1)), r(1 - F(_pow_exact(f32(beta_2), f32(t))))
