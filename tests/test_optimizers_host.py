"""Host-side tests of the RMSprop, Adadelta and Adamax optimizers: the oracle's rules against two-step closed forms, the
facade's per-table semantics, optimizers.get, the slot layout and the refusals."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

import optim_oracle
from ampligraph_b200 import _lib
from ampligraph_b200.latent_features import optimizers

X0 = np.array([0.5, -0.25, 0.125, 0.0, -1.0], np.float64)
G1 = np.array([0.1, -0.3, 0.0, 2.0, 0.05], np.float64)
G2 = np.array([-0.2, -0.1, 0.0, 1.0, 0.4], np.float64)


def _oracle_two_steps(name, lr, hp):
    x = torch.tensor(X0, dtype=torch.float32)
    a, b = torch.zeros_like(x), torch.zeros_like(x)
    for t, g in ((1, G1), (2, G2)):
        optim_oracle.rule(name, x, torch.tensor(g, dtype=torch.float32), a, b, t, lr, hp)
    return x.numpy().astype(np.float64), a.numpy().astype(np.float64), b.numpy().astype(np.float64)


def _closed_form(name, lr, hp):
    """the textbook recursions in fp64"""
    eps = hp.get("epsilon", 1e-7)
    x, a, b = X0.copy(), np.zeros_like(X0), np.zeros_like(X0)
    for t, g in ((1, G1), (2, G2)):
        if name == "rmsprop":
            rho, mu = hp.get("rho", 0.9), hp.get("momentum", 0.0)
            a = rho * a + (1 - rho) * g * g
            if mu:
                b = mu * b + lr * g / np.sqrt(a + eps)
                x = x - b
            else:
                d = a
                if hp.get("centered"):
                    b = rho * b + (1 - rho) * g
                    d = a - b * b
                x = x - lr * g / (np.sqrt(d) + eps)
        elif name == "adadelta":
            rho = hp.get("rho", 0.95)
            a = rho * a + (1 - rho) * g * g
            u = np.sqrt(b + eps) / np.sqrt(a + eps) * g
            x = x - lr * u
            b = rho * b + (1 - rho) * u * u
        else:
            b1, b2 = hp.get("beta_1", 0.9), hp.get("beta_2", 0.999)
            a = b1 * a + (1 - b1) * g
            b = np.maximum(b2 * b, np.abs(g))
            x = x - lr / (1 - b1 ** t) * a / (b + eps)
    return x, a, b


@pytest.mark.parametrize("name,lr,hp", [
    ("rmsprop", 0.01, {}), ("rmsprop", 0.01, {"rho": 0.8, "centered": True}),
    ("rmsprop", 0.01, {"momentum": 0.9}), ("rmsprop", 0.05, {"rho": 0.7, "momentum": 0.5, "epsilon": 1e-3}),
    ("adadelta", 1.0, {}), ("adadelta", 0.5, {"rho": 0.9, "epsilon": 1e-6}),
    ("adamax", 0.01, {}), ("adamax", 0.002, {"beta_1": 0.8, "beta_2": 0.99})])
def test_oracle_rules_two_step_closed_form(name, lr, hp):
    got, want = _oracle_two_steps(name, lr, hp), _closed_form(name, lr, hp)
    for g, w in zip(got, want):
        assert np.allclose(g, w, rtol=2e-6, atol=1e-7), (g, w)


def test_oracle_refuses_centered_rmsprop_with_momentum():
    x = torch.zeros(3)
    with pytest.raises(NotImplementedError):
        optim_oracle.rule("rmsprop", x, x, x.clone(), x.clone(), 1, 0.01, {"momentum": 0.9, "centered": True})


def test_oracle_lazy_rule_moves_only_listed_rows():
    """The looked-up-rows restatement: listed rows take the dense rule (even with a zero gradient), the rest keep their
    value and their slots."""
    var = torch.tensor([[1.0, 2.0], [3.0, 4.0], [5.0, 6.0]])
    grad = torch.tensor([[0.5, -0.5], [0.0, 0.0], [1.0, 1.0]])
    opt = optim_oracle.Optimizer("adamax", 0.1, lazy_tables={"ent": True})
    dense = optim_oracle.Optimizer("adamax", 0.1)
    v2 = var.clone()
    opt.step({"ent": (var, grad)}, {"ent": torch.tensor([0, 1, 0])})
    dense.step({"ent": (v2, grad.clone())})
    assert torch.equal(var[:2], v2[:2]) and torch.equal(var[2], torch.tensor([5.0, 6.0]))
    assert (opt.slots["ent"][0][2] == 0).all() and (opt.slots["ent"][0][0] != 0).all()


@pytest.mark.parametrize("name,hp,regularized,want", [
    ("adam", {}, (False, False), (False, False)),
    ("sgd", {"momentum": 0.9}, (False, False), (False, False)),
    ("adagrad", {}, (False, True), (False, False)),
    ("rmsprop", {}, (False, False), (False, False)),
    ("rmsprop", {"centered": True}, (False, False), (False, False)),
    ("rmsprop", {"momentum": 0.9}, (False, False), (True, True)),
    ("rmsprop", {"momentum": 0.9}, (True, False), (False, True)),
    ("rmsprop", {"momentum": 0.9}, (True, True), (False, False)),
    ("adadelta", {}, (False, False), (False, False)),
    ("adamax", {}, (False, False), (True, True)),
    ("adamax", {}, (True, False), (False, True)),
    ("adamax", {}, (False, True), (True, False)),
    ("adamax", {}, (True, True), (False, False)),
    ("lazy_adadelta", {}, (True, True), (True, True)),
    ("lazy_adam", {}, (False, False), (True, True)),
    ("RMSprop", {"momentum": 0.5}, (False, True), (True, False))])
def test_table_rules(name, hp, regularized, want):
    assert optimizers.table_rules(name, hp, regularized) == want


def test_get_by_name_and_by_config_object():
    for name in ("rmsprop", "adadelta", "adamax", "lazy_rmsprop", "lazy_adadelta", "lazy_adamax"):
        w = optimizers.get(name, {"learning_rate": 0.01})
        assert w.name == name and w.hyperparams["learning_rate"] == 0.01 and w.get_hyperparam_count() == 1
    assert optimizers.get("adamax").hyperparams == {"learning_rate": 0.001}

    class RMSprop:  # what a Keras legacy optimizer's get_config() returns
        def get_config(self):
            return {"name": "RMSprop", "learning_rate": 0.002, "decay": 0.0, "rho": 0.8, "momentum": 0.0,
                    "epsilon": 1e-6, "centered": True}

    class Adadelta:
        def get_config(self):
            return {"name": "Adadelta", "learning_rate": 1.0, "rho": 0.9, "epsilon": 1e-7}

    w = optimizers.get(RMSprop())
    assert w.name == "rmsprop"
    assert w.hyperparams == {"learning_rate": 0.002, "rho": 0.8, "momentum": 0.0, "epsilon": 1e-6, "centered": True}
    w = optimizers.get(Adadelta())
    assert w.name == "adadelta" and w.hyperparams == {"learning_rate": 1.0, "rho": 0.9, "epsilon": 1e-7}
    for bad in ("nadam", "ftrl", "lazy_nadam"):
        with pytest.raises(ValueError):
            optimizers.get(bad)


def _cfg(name, **kw):
    c = _lib.KgeOptimizerConfig(C.sizeof(_lib.KgeOptimizerConfig), _lib.OPTIMIZERS[name])
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def test_optimizer_slots():
    from ampligraph_b200.engine import optimizer_slots
    assert optimizer_slots(_cfg("sgd")) == (None, None)
    assert optimizer_slots(_cfg("sgd", momentum=0.9)) == (0.0, None)
    assert optimizer_slots(_cfg("adam")) == (0.0, 0.0)
    assert optimizer_slots(_cfg("adagrad", initial_accumulator_value=0.25)) == (0.25, None)
    assert optimizer_slots(_cfg("rmsprop")) == (0.0, None)
    assert optimizer_slots(_cfg("rmsprop", centered=1)) == (0.0, 0.0)
    assert optimizer_slots(_cfg("rmsprop", momentum=0.5)) == (0.0, 0.0)
    assert optimizer_slots(_cfg("adadelta")) == (0.0, 0.0)
    assert optimizer_slots(_cfg("adamax")) == (0.0, 0.0)


def test_config_layout_keeps_the_old_prefix(tmp_path):
    """The new fields are appended: the old layout is the prefix up to rho, and the enum values are the binding's."""
    src = tmp_path / "o.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "%s"\nint main(void){printf("%%zu %%zu %%zu %%d %%d %%d",'
                   'offsetof(kge_optimizer_config, rho), offsetof(kge_optimizer_config, centered), '
                   'sizeof(kge_optimizer_config), KGE_OPT_RMSPROP, KGE_OPT_ADADELTA, KGE_OPT_ADAMAX); return 0;}' % _lib.HEADER)
    exe = tmp_path / "o"
    subprocess.run(["cc", "-o", str(exe), str(src)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    K = _lib.KgeOptimizerConfig
    assert got == [48, K.centered.offset, C.sizeof(K), _lib.OPTIMIZERS["rmsprop"], _lib.OPTIMIZERS["adadelta"],
                   _lib.OPTIMIZERS["adamax"]]
    assert K.rho.offset == 48 and K.reg_lambda2.offset + 4 == 48


def test_lazy_tables_refused_under_replicated_training():
    from ampligraph_b200.parallel import reject_lazy
    for name in ("lazy_rmsprop", "lazy_adadelta", "lazy_adamax"):
        reject_lazy(name, 1)
        with pytest.raises(NotImplementedError):
            reject_lazy(name, 2)
    reject_lazy("adamax", 4)
