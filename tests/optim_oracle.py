"""Restatement of the RMSprop, Adadelta and Adamax rules (TF 2.15 legacy Keras optimizers and the training ops they
call) in the fp32 operation order of kge_optim_common.cuh, on top of oracle.ref_step, plus the reference's per-table
choice between the dense rule and the looked-up-rows rule (a regulariser per table).  TensorFlow cannot be installed
here, so, like the other rules of oracle.ref_step, these follow the documented semantics and are not pinned by a TF run.
Test infrastructure only: tests and __graft_entry__.smoke() import it."""
import numpy as np
import torch

from oracle import ref_step
from optim_exact_oracle import fma32

NEW_KINDS = ("rmsprop", "adadelta", "adamax")
RHO_DEFAULT = {"rmsprop": 0.9, "adadelta": 0.95}
f32 = np.float32


def _fma(a, b, c):
    """fp32 fma(a, b, c), correctly rounded (optim_exact_oracle.fma32), as an fp32 tensor."""
    n = lambda v: v.detach().cpu().numpy() if torch.is_tensor(v) else v
    return torch.from_numpy(np.ascontiguousarray(fma32(n(a), n(b), n(c))))


def rule(name, x, g, a, b, t, lr, hp):
    """One step of kind `name` on fp32 tensors: x, a (slot 0), b (slot 1) updated in place, g the summed gradient."""
    lr = f32(lr)
    eps = f32(hp.get("epsilon", 1e-7))
    if name == "rmsprop":
        rho, mu = f32(hp.get("rho", 0.9)), f32(hp.get("momentum", 0.0))
        g2, step = g * g, lr * g
        if mu != 0:
            if hp.get("centered"):
                raise NotImplementedError("centered RMSprop with momentum")
            a.copy_(_fma(g2 - a, f32(1) - rho, a))
            b.copy_(_fma(mu, b, step / torch.sqrt(a + eps)))
            x.sub_(b)
        else:
            a.copy_(_fma(rho, a, (f32(1) - rho) * g2))
            d = a
            if hp.get("centered"):
                b.copy_(_fma(rho, b, (f32(1) - rho) * g))
                d = _fma(-b, b, a)
            x.sub_(step / (torch.sqrt(d) + eps))
    elif name == "adadelta":
        rho = f32(hp.get("rho", 0.95))
        a.copy_(_fma(rho, a, (f32(1) - rho) * (g * g)))
        u = (torch.sqrt(b + eps) / torch.sqrt(a + eps)) * g
        x.copy_(_fma(-lr, u, x))
        b.copy_(_fma(rho, b, (f32(1) - rho) * (u * u)))
    elif name == "adamax":
        b1, b2 = f32(hp.get("beta_1", 0.9)), f32(hp.get("beta_2", 0.999))
        lr_t = f32(float(lr) / (1.0 - float(b1) ** t))  # fp64 on the host, rounded once
        a.copy_(_fma(g - a, f32(1) - b1, a))
        b.copy_(torch.maximum(b2 * b, g.abs()))
        x.copy_(_fma(-lr_t, a / (b + eps), x))
    else:
        raise ValueError(name)


class Optimizer(ref_step.LegacyOptimizer):
    """ref_step.LegacyOptimizer with the three rules above, and the looked-up-rows rule chosen per table:
    lazy_tables = {key: bool} (default: the 'lazy_' prefix for every table).  Slots start at 0."""

    def __init__(self, name="adam", learning_rate=0.001, lazy_tables=None, **hp):
        super().__init__(name, learning_rate, **hp)
        self.lazy_tables = lazy_tables

    def _slots(self, key, like):
        if self.name in NEW_KINDS:
            return self.slots.setdefault(key, (torch.zeros_like(like), torch.zeros_like(like)))
        return None

    def apply(self, var, grad, key):
        if self.name not in NEW_KINDS:
            return super().apply(var, grad, key)
        a, b = self._slots(key, var)
        rule(self.name, var, grad, a, b, self.t, self.lr, self.hp)

    def step(self, named_vars_grads, touched=None):
        if self.name not in NEW_KINDS and self.lazy_tables is None:
            return super().step(named_vars_grads, touched)
        self.t += 1
        for key, (var, grad) in named_vars_grads.items():
            lazy = self.lazy if self.lazy_tables is None else self.lazy_tables[key]
            if not lazy:
                self.apply(var, grad, key)
                continue
            if self.name not in NEW_KINDS:
                raise NotImplementedError("per-table choice is restated for %s only" % (NEW_KINDS,))
            rows = torch.unique(touched[key])
            a, b = self._slots(key, var)
            sub, sa, sb = var[rows].clone(), a[rows].clone(), b[rows].clone()
            rule(self.name, sub, grad[rows], sa, sb, self.t, self.lr, self.hp)
            var[rows], a[rows], b[rows] = sub, sa, sb


class RefStep(ref_step.RefStep):
    """ref_step.RefStep with Optimizer, a regulariser per table (regularizer: None, one dict for both tables, or a
    pair [entities, relations]) and lazy_tables as in Optimizer."""

    def __init__(self, model, K, ent, rel, eta, loss="pairwise", loss_params=None, optimizer="adam",
                 optimizer_params=None, regularizer=None, lazy_tables=None):
        super().__init__(model, K, ent, rel, eta, loss, loss_params, optimizer, optimizer_params, None)
        op = dict(optimizer_params or {})
        self.opt = Optimizer(optimizer, op.pop("learning_rate", 0.001), lazy_tables=lazy_tables, **op)
        self.regs = list(regularizer) if isinstance(regularizer, (list, tuple)) else [regularizer, regularizer]

    def loss_and_grads(self, triples, corruptions):
        for v in (self.ent, self.rel):
            v.grad = None
        sp, sn = self.forward(triples, corruptions)
        regs = [ref_step.lp_regularizer(v, r.get("lam", 1e-5), r.get("p", 2)) for v, r in zip((self.ent, self.rel), self.regs)
                if r]
        loss = ref_step.total_loss(self.loss, sp, sn, self.eta, regs, **self.loss_params)
        loss.backward()
        return loss.detach(), sp.detach(), sn.detach(), self.ent.grad, self.rel.grad

    def train_step(self, triples, corruptions):
        loss, sp, sn, g_ent, g_rel = self.loss_and_grads(triples, corruptions)
        with torch.no_grad():
            t = torch.as_tensor(triples, dtype=torch.long)
            c = torch.as_tensor(corruptions, dtype=torch.long)
            touched = {"ent": torch.cat([t[:, 0], t[:, 2], c[:, 0], c[:, 2]]), "rel": t[:, 1]}
            self.opt.step({"ent": (self.ent, g_ent), "rel": (self.rel, g_rel)}, touched)
        return float(loss)
