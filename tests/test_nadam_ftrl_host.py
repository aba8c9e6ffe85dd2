"""Host-side tests of the Nadam and Ftrl optimizers: name, wrapper and Keras-config resolution, the per-table rules,
Nadam's fp32 per-step scalars against an exact restatement, the restatement of both rules against fp64 closed forms (Ftrl zeroing the
rows a first step does not touch included), the slots and the C config's layouts."""
import ctypes as C
import subprocess

import numpy as np
import pytest

import nadam_ftrl_oracle as nfo
from ampligraph_b200 import _lib
from ampligraph_b200.engine import nadam_coefficients, optimizer_slots
from ampligraph_b200.latent_features import optimizers

f32 = np.float32


def test_names_and_keras_configs():
    assert optimizers.KINDS[-2:] == ("nadam", "ftrl")
    assert [_lib.OPTIMIZERS[k] for k in optimizers.KINDS] == list(range(8))
    for name in ("nadam", "ftrl", "lazy_nadam", "lazy_ftrl", "Nadam"):
        w = optimizers.OptimizerWrapper(name, {"learning_rate": 0.01})
        assert w.name == name.lower() and w.hyperparams == {"learning_rate": 0.01}
        assert w.get_hyperparam_count() == 1  # Nadam is not one of the reference's Adam classes
        assert optimizers.get(w) is w
        with pytest.raises(ValueError):  # a name string resolves to the six older kinds only (optimizers.NAMES)
            optimizers.get(name)
    assert optimizers.get("adam").get_hyperparam_count() == 2
    assert set(optimizers.NAMES) == {k for k in optimizers.SUPPORTED if "nadam" not in k and "ftrl" not in k}
    for bad in ("adamw", "lazy_adamw", "nag", "lazy_"):
        with pytest.raises(ValueError):
            optimizers.OptimizerWrapper(bad)

    class Nadam:  # Keras' legacy Nadam stores schedule_decay as `decay`
        def get_config(self):
            return {"name": "Nadam", "learning_rate": 0.002, "decay": 0.004, "beta_1": 0.9, "beta_2": 0.999,
                    "epsilon": 1e-7}

    class Ftrl:
        def get_config(self):
            return {"name": "Ftrl", "learning_rate": 0.05, "decay": 0.0, "initial_accumulator_value": 0.2,
                    "learning_rate_power": -0.75, "l1_regularization_strength": 0.01,
                    "l2_regularization_strength": 0.02, "l2_shrinkage_regularization_strength": 0.03, "beta": 0.5}

    w = optimizers.get(Nadam())
    assert w.name == "nadam"
    assert w.hyperparams == {"learning_rate": 0.002, "decay": 0.004, "beta_1": 0.9, "beta_2": 0.999, "epsilon": 1e-7}
    w = optimizers.get(Ftrl())
    assert w.name == "ftrl"
    assert w.hyperparams == {"learning_rate": 0.05, "initial_accumulator_value": 0.2, "learning_rate_power": -0.75,
                             "l1_regularization_strength": 0.01, "l2_regularization_strength": 0.02,
                             "l2_shrinkage_regularization_strength": 0.03, "beta": 0.5}


@pytest.mark.parametrize("name,hp,regularized,want", [
    ("nadam", {}, (False, False), (True, True)),
    ("nadam", {}, (True, False), (False, True)),
    ("nadam", {}, (False, True), (True, False)),
    ("Nadam", {}, (True, True), (False, False)),
    ("ftrl", {}, (False, False), (False, False)),
    ("ftrl", {"l1_regularization_strength": 0.1}, (True, False), (False, False)),
    ("lazy_nadam", {}, (True, False), (True, True)),
    ("lazy_ftrl", {}, (False, False), (True, True))])
def test_table_rules(name, hp, regularized, want):
    assert optimizers.table_rules(name, hp, regularized) == want


def _cfg(name, **kw):
    c = _lib.KgeOptimizerConfig(C.sizeof(_lib.KgeOptimizerConfig), _lib.OPTIMIZERS[name])
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def test_optimizer_slots():
    assert optimizer_slots(_cfg("nadam")) == (0.0, 0.0)
    assert optimizer_slots(_cfg("ftrl", initial_accumulator_value=0.25)) == (0.25, 0.0)
    assert optimizer_slots(_cfg("ftrl", initial_accumulator_value=0.0)) == (0.0, 0.0)


def _bits(v):
    return np.asarray(v, f32).view(np.uint32)


@pytest.mark.parametrize("b1,b2,decay", [(0.9, 0.999, 0.004), (0.5, 0.9, 0.1), (0.99, 0.9999, 0.0)])
def test_nadam_coefficients_1000_steps(b1, b2, decay):
    """engine.nadam_coefficients, chained through its own cache for 1,000 steps (the cache underflows to subnormals and
    to 0 on the way), equals the exact rational restatement bit for bit at every step."""
    c, ce = f32(1.0), f32(1.0)
    for t in range(1, 1001):
        got = nadam_coefficients(b1, b2, decay, t, c)
        want = nfo.nadam_coefficients_exact(b1, b2, decay, t, ce)
        assert all(isinstance(v, np.float32) for v in got)
        assert (_bits(got) == _bits(want)).all(), (t, got, want)
        c, ce = got[2], want[2]
    if decay > 0:
        assert c == 0.0  # s_new is a product of ~0.5 factors


def _nadam_cfg(t, cache, **kw):
    c = _cfg("nadam", learning_rate=0.01, beta_1=0.9, beta_2=0.999, epsilon=1e-7, **kw)
    c.nadam_m_t, c.nadam_m_t1, c.nadam_s_new, c.nadam_s_next, c.nadam_v_den = nadam_coefficients(
        c.beta_1, c.beta_2, 0.004, t, cache)
    return c


def test_oracle_nadam_against_fp64():
    """Two steps of the restatement against Keras' formulas in fp64 (the same per-step scalars), within a few fp32
    rounding errors; the row-decay mode: a decayed row keeps x and scales m, v by b1, b2 exactly, a looked-up row with
    an exactly zero gradient still moves."""
    rng = np.random.default_rng(0)
    x = rng.uniform(-1, 1, 64).astype(f32)
    g1, g2 = (rng.uniform(-1, 1, 64).astype(f32) for _ in range(2))
    a = b = np.zeros(64, f32)
    xd, ad, bd = (v.astype(np.float64) for v in (x, a, b))
    cache = f32(1.0)
    for t, g in ((1, g1), (2, g2)):
        cfg = _nadam_cfg(t, cache)
        cache = f32(cfg.nadam_s_new)
        x, a, b = nfo.update(cfg, t, x, g, a, b)
        gd = g.astype(np.float64)
        b1, b2 = float(f32(0.9)), float(f32(0.999))
        ad = b1 * ad + (1 - b1) * gd
        bd = b2 * bd + (1 - b2) * gd * gd
        mb = (1 - float(cfg.nadam_m_t)) * gd / (1 - float(cfg.nadam_s_new)) + float(cfg.nadam_m_t1) * ad / (
            1 - float(cfg.nadam_s_next))
        xd = xd - float(f32(0.01)) * mb / (np.sqrt(bd / float(cfg.nadam_v_den)) + float(f32(1e-7)))
    assert np.allclose(x, xd, rtol=1e-5, atol=1e-6) and np.allclose(a, ad, rtol=1e-5, atol=1e-7)
    assert np.allclose(b, bd, rtol=1e-5, atol=1e-9)

    cfg = _nadam_cfg(3, cache)
    m0 = np.array([0.5, -0.25, 0.0, 3.0], f32)
    v0 = np.array([0.25, 1.0, 0.5, 0.0], f32)
    x0 = np.array([1.0, 2.0, -3.0, 4.0], f32)
    g0 = np.zeros(4, f32)
    moved = np.array([False, True, False, True])
    nx, na, nb = nfo.update(cfg, 3, x0, g0, m0, v0, moved=moved)
    assert (nx[~moved] == x0[~moved]).all()  # not looked up: no move even with m != 0
    assert (_bits(na[~moved]) == _bits(f32(0.9) * m0[~moved])).all()
    assert (_bits(nb[~moved]) == _bits(f32(0.999) * v0[~moved])).all()
    assert nx[1] != x0[1]  # looked up, gradient exactly 0, m != 0: moves


def _ftrl_fp64(x, g, n, z, lr, p, l1, l2, shrink, beta):
    l2a = l2 + beta / (2 * lr)
    gs = g + 2 * shrink * x
    n1 = n + g * g
    z = z + gs - (n1 ** -p - n ** -p) / lr * x
    q = n1 ** -p / lr + 2 * l2a
    x = np.where(np.abs(z) > l1, (np.sign(z) * l1 - z) / q, 0.0)
    return x, n1, z


@pytest.mark.parametrize("hp", [dict(lr_power=-0.5), dict(lr_power=-0.25, l1=0.01), dict(lr_power=-0.5, l2=0.1, ftrl_beta=0.5),
                                dict(lr_power=-0.5, l2_shrinkage=0.2, l1=0.001), dict(lr_power=-1.5, l2=0.01)])
def test_oracle_ftrl_against_fp64(hp):
    """Two steps of the restatement (ApplyFtrl / ApplyFtrlV2, the sqrt and the pow path, l1, l2, beta, shrinkage)
    against the same formulas in fp64."""
    rng = np.random.default_rng(1)
    cfg = _cfg("ftrl", learning_rate=0.05, **hp)
    x = rng.uniform(-1, 1, 64).astype(f32)
    n = np.full(64, 0.1, f32)
    z = np.zeros(64, f32)
    xd, nd, zd = (v.astype(np.float64) for v in (x, n, z))
    for _ in range(2):
        g = rng.uniform(-1, 1, 64).astype(f32)
        x, n, z = nfo.update(cfg, 1, x, g, n, z)
        xd, nd, zd = _ftrl_fp64(xd, g.astype(np.float64), nd, zd, float(f32(0.05)), float(f32(cfg.lr_power)),
                                float(f32(cfg.l1)), float(f32(cfg.l2)), float(f32(cfg.l2_shrinkage)),
                                float(f32(cfg.ftrl_beta)))
    assert np.allclose(x, xd, rtol=1e-4, atol=1e-6) and np.allclose(n, nd, rtol=1e-6)
    assert np.allclose(z, zd, rtol=1e-4, atol=1e-6)


def test_oracle_ftrl_zeroes_untouched_rows_on_step_1():
    """The dense rule on a row without a gradient at step 1: z stays 0, |z| > l1 is false, x becomes 0 -- what the
    reference does to every row a first step does not look up.  |z| == l1 exactly does not move x off 0 either."""
    cfg = _cfg("ftrl", learning_rate=0.05, lr_power=-0.5, l1=0.5)
    x = np.array([0.3, -2.0, 1e-20, 0.0], f32)
    nx, n, z = nfo.update(cfg, 1, x, np.zeros(4, f32), np.full(4, 0.1, f32), np.zeros(4, f32))
    assert (_bits(nx) == 0).all() and (z == 0).all() and (n == f32(0.1)).all()
    nx, _, z = nfo.update(cfg, 1, np.zeros(3, f32), np.zeros(3, f32), np.full(3, 0.1, f32),
                          np.array([0.5, -0.5, np.nextafter(f32(0.5), f32(1))], f32))
    assert nx[0] == 0 and nx[1] == 0 and nx[2] < 0  # |z| == l1: 0; just above: moves against z


def test_config_layouts(tmp_path):
    """The Nadam and Ftrl fields are appended: the layout before RMSprop stops at rho (48 bytes), the layout before Nadam
    and Ftrl at l1 (56 bytes); the enum values are the binding's."""
    src = tmp_path / "o.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "%s"\nint main(void){printf("%%zu %%zu %%zu %%zu '
                   '%%d %%d",offsetof(kge_optimizer_config, rho), offsetof(kge_optimizer_config, l1), '
                   'offsetof(kge_optimizer_config, nadam_v_den), sizeof(kge_optimizer_config), KGE_OPT_NADAM, '
                   'KGE_OPT_FTRL); return 0;}' % _lib.HEADER)
    exe = tmp_path / "o"
    subprocess.run(["cc", "-o", str(exe), str(src)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    K = _lib.KgeOptimizerConfig
    assert got == [48, 56, K.nadam_v_den.offset, C.sizeof(K), _lib.OPTIMIZERS["nadam"], _lib.OPTIMIZERS["ftrl"]]
    assert K.l1.offset == 56 and K.centered.offset + 4 == 56 and C.sizeof(K) == 96
