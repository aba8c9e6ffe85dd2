"""ref_step.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Torch-CPU fp32 restatement, op for op, of the reference's *training step*
(lookup -> corrupt -> score -> loss -> tape.gradient -> optimizer) so that the
CUDA path has something to be checked against and timed beside.  TensorFlow is
not installable in this image (python 3.12, no wheel), hence torch autograd
stands in for tf.GradientTape; every function cites the reference lines it
follows (paths under ampligraph/latent_features/ of the reference).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
--impl reference legs may import this module.

Parity status
  * scoring functions, losses, lookup: PINNED by the reference's own golden
    vectors (tests/golden/reference_kats.json; tests/test_oracle.py).
  * optimizer arithmetic (TF legacy Adam/SGD/Adagrad kernels), Glorot stream,
    corruption RNG stream: the arithmetic lives in TensorFlow, which is not
    vendored; the reference's tests pin none of it.  PARITY UNPINNED -- this
    file follows the documented TF 2.15 legacy semantics and is itself the pin.
"""
import math

import numpy as np
import torch

CLIP_LO, CLIP_HI = -75.0, 75.0  # loss_functions.py:32-35


# --------------------------------------------------------------------------
# scoring: layers/scoring/*.py  (_compute_scores on gathered [n,K] rows)
# --------------------------------------------------------------------------
def rotate_divisor(K, max_rel_size):
    """RotatE.py:96-98: theta / (embedding_range / pi)."""
    rng = (6.0 / (K * max_rel_size)) ** 0.5
    return rng / math.pi


def compute_scores(model, e_s, e_p, e_o, max_rel_size=None):
    K = e_s.shape[1]
    h = K // 2
    if model == "TransE":  # TransE.py:51-53
        return -torch.sum(torch.abs(e_s + e_p - e_o), dim=1)
    if model == "DistMult":  # DistMult.py:48
        return torch.sum(e_s * e_p * e_o, dim=1)
    if model in ("ComplEx", "HolE"):  # ComplEx.py:52-62, HolE.py:45
        s_re, s_im = e_s[:, :h], e_s[:, h:]
        p_re, p_im = e_p[:, :h], e_p[:, h:]
        o_re, o_im = e_o[:, :h], e_o[:, h:]
        sc = torch.sum(s_re * (p_re * o_re + p_im * o_im) + s_im * (p_re * o_im - p_im * o_re), dim=1)
        if model == "HolE":
            sc = (2.0 / (K / 2.0)) * sc
        return sc
    if model == "RotatE":  # RotatE.py:76-104
        s_re, s_im = e_s[:, :h], e_s[:, h:]
        o_re, o_im = e_o[:, :h], e_o[:, h:]
        theta = e_p[:, :h]
        div = rotate_divisor(K, max_rel_size if max_rel_size else 1)
        p_re, p_im = torch.cos(theta / div), torch.sin(theta / div)
        re = s_re * p_re - s_im * p_im - o_re
        im = s_re * p_im + s_im * p_re - o_im
        return -torch.sum(torch.sqrt(re ** 2 + im ** 2), dim=1)
    raise ValueError(model)


def corruption_scores(model, side, e_s, e_p, e_o, ent_matrix, max_rel_size=None):
    """_get_subject_corruption_scores / _get_object_corruption_scores: the
    broadcast [b, m, K] form the reference uses."""
    K = e_s.shape[1]
    h = K // 2
    E = ent_matrix.unsqueeze(0)  # [1,m,K]
    if model == "TransE":  # TransE.py:78-84, :107-113
        if side == "s":
            return -torch.sum(torch.abs(E + (e_p - e_o).unsqueeze(1)), dim=2)
        return -torch.sum(torch.abs((e_s + e_p).unsqueeze(1) - E), dim=2)
    if model == "DistMult":  # DistMult.py:71-73, :96-98
        if side == "s":
            return torch.sum(E * (e_p * e_o).unsqueeze(1), dim=2)
        return torch.sum((e_s * e_p).unsqueeze(1) * E, dim=2)
    if model in ("ComplEx", "HolE"):
        s_re, s_im = e_s[:, :h], e_s[:, h:]
        p_re, p_im = e_p[:, :h], e_p[:, h:]
        o_re, o_im = e_o[:, :h], e_o[:, h:]
        e_re, e_im = E[:, :, :h], E[:, :, h:]
        if side == "s":  # ComplEx.py:95-108
            sc = torch.sum(e_re * ((p_re * o_re).unsqueeze(1) + (p_im * o_im).unsqueeze(1))
                           + e_im * ((p_re * o_im).unsqueeze(1) - (p_im * o_re).unsqueeze(1)), dim=2)
        else:  # ComplEx.py:139-150
            sc = torch.sum(((s_re * p_re).unsqueeze(1) - (s_im * p_im).unsqueeze(1)) * e_re
                           + ((s_im * p_re).unsqueeze(1) + (s_re * p_im).unsqueeze(1)) * e_im, dim=2)
        if model == "HolE":
            sc = (2.0 / (K / 2.0)) * sc
        return sc
    if model == "RotatE":
        s_re, s_im = e_s[:, :h], e_s[:, h:]
        o_re, o_im = e_o[:, :h], e_o[:, h:]
        theta = e_p[:, :h]
        div = rotate_divisor(K, max_rel_size if max_rel_size else 1)
        p_re, p_im = torch.cos(theta / div), torch.sin(theta / div)
        e_re, e_im = E[:, :, :h], E[:, :, h:]
        if side == "s":  # RotatE.py:151-163
            re = e_re * p_re.unsqueeze(1) - e_im * p_im.unsqueeze(1) - o_re.unsqueeze(1)
            im = e_re * p_im.unsqueeze(1) + e_im * p_re.unsqueeze(1) - o_im.unsqueeze(1)
        else:  # RotatE.py:208-216
            re = (s_re * p_re - s_im * p_im).unsqueeze(1) - e_re
            im = (s_re * p_im + s_im * p_re).unsqueeze(1) - e_im
        return -torch.sum(torch.sqrt(re ** 2 + im ** 2), dim=2)
    raise ValueError(model)


# --------------------------------------------------------------------------
# losses: loss_functions.py
# --------------------------------------------------------------------------
def _reduce(x, reduction):  # loss_functions.py:124-129
    return x.sum(0) if reduction == "sum" else x.mean(0)


def per_positive_loss(name, scores_pos, scores_neg, margin=None, alpha=None, reduction="sum"):
    """_apply_loss of each loss; scores_neg is [eta, B] (loss_functions.py:211)."""
    if name == "pairwise":  # :286-308
        m = 1.0 if margin is None else margin
        return _reduce(torch.clamp(m - scores_pos + scores_neg, min=0), reduction)
    if name == "nll":  # :360-382
        sn = torch.clamp(scores_neg, CLIP_LO, CLIP_HI)
        sp = torch.clamp(scores_pos, CLIP_LO, CLIP_HI)
        sp = sp.repeat(sn.shape[0]).reshape(sn.shape[0], -1)  # _broadcast_score_pos :165-183
        sc = torch.cat([-sp, sn], 0)
        return _reduce(torch.log(1 + torch.exp(sc)), reduction)
    if name == "absolute_margin":  # :442-464
        m = 1.0 if margin is None else margin
        return _reduce(torch.clamp(m + scores_neg, min=0) - scores_pos, reduction)
    if name == "self_adversarial":  # :540-574 (no stop-gradient on p_neg)
        m = 3.0 if margin is None else margin
        a = 0.5 if alpha is None else alpha
        p_neg = torch.softmax(a * scores_neg, dim=0)
        return -torch.nn.functional.logsigmoid(m + scores_pos) - _reduce(
            p_neg * torch.nn.functional.logsigmoid(-scores_neg - m), reduction)
    if name == "multiclass_nll":  # :630-654
        sp = torch.clamp(scores_pos, CLIP_LO, CLIP_HI)
        sn = torch.clamp(scores_neg, CLIP_LO, CLIP_HI)
        neg_exp, pos_exp = torch.exp(sn), torch.exp(sp)
        return -torch.log(pos_exp / (_reduce(neg_exp, reduction) + pos_exp))
    raise ValueError("Could not interpret loss identifier: %s" % name)  # :757


def total_loss(name, scores_pos, scores_neg_flat, eta, reg_losses=(), **kw):
    """Loss.__call__ :185-225: reshape to [eta,-1], SUM over the batch, add regularisers."""
    sn = scores_neg_flat.reshape(eta, -1)
    loss = per_positive_loss(name, scores_pos, sn, **kw).sum()
    for r in reg_losses:
        loss = loss + r
    return loss


def lp_regularizer(x, lam=1e-5, p=2):  # regularizers.py:14-37
    return lam * torch.sum(torch.abs(x) ** p)


# --------------------------------------------------------------------------
# corruption structure: CorruptionGenerationLayerTrain.py:52-94
# --------------------------------------------------------------------------
def corrupt(pos, eta, keep_subj, repl):
    """pos [B,3] int; keep_subj, repl [eta*B]; row j*B+i = j-th corruption of i."""
    ds = pos.repeat(eta, 1)  # tf.tile(pos,[eta,1])
    ks = keep_subj.to(ds.dtype)
    ko = 1 - ks
    subj = ks * ds[:, 0] + ko * repl
    obj = ko * ds[:, 2] + ks * repl
    return torch.stack([subj, ds[:, 1], obj], dim=1)


# --------------------------------------------------------------------------
# optimizers (TF 2.15 tf.keras.optimizers.legacy.*; optimizers.py:255-291)
# --------------------------------------------------------------------------
class LegacyOptimizer:
    """Dense-semantics restatement: legacy Keras sums duplicate IndexedSlices
    rows first, then Adam decays m/v for EVERY row and moves every row."""

    def __init__(self, name="adam", learning_rate=0.001, **hp):
        # 'lazy_<name>': update only rows with a gradient contribution this step (the documented
        # semantics of TensorFlow-Addons LazyAdam; NOT the reference's rule -- an extension of the product)
        self.lazy = name.lower().startswith("lazy_")
        name = name.lower()[5:] if self.lazy else name
        self.name = name.lower()
        self.lr = float(learning_rate)
        self.hp = hp
        self.t = 0
        self.slots = {}

    def apply(self, var, grad, key):
        f32 = np.float32
        if self.name == "sgd":
            mom = float(self.hp.get("momentum", 0.0))
            if mom == 0.0:
                var.sub_(f32(self.lr) * grad)
            else:
                acc = self.slots.setdefault(key, torch.zeros_like(var))
                acc.mul_(f32(mom)).sub_(f32(self.lr) * grad)
                var.add_(acc)
        elif self.name == "adam":
            b1 = float(self.hp.get("beta_1", 0.9))
            b2 = float(self.hp.get("beta_2", 0.999))
            eps = float(self.hp.get("epsilon", 1e-7))
            m, v = self.slots.setdefault(key, (torch.zeros_like(var), torch.zeros_like(var)))
            lr_t = self.lr * math.sqrt(1.0 - b2 ** self.t) / (1.0 - b1 ** self.t)
            m.mul_(f32(b1)).add_(grad * f32(1.0 - b1))
            v.mul_(f32(b2)).add_(grad * grad * f32(1.0 - b2))
            var.sub_(f32(lr_t) * m / (torch.sqrt(v) + f32(eps)))
        elif self.name == "adagrad":
            eps = float(self.hp.get("epsilon", 1e-7))
            init = float(self.hp.get("initial_accumulator_value", 0.1))
            acc = self.slots.setdefault(key, torch.full_like(var, init))
            acc.add_(grad * grad)
            var.sub_(f32(self.lr) * grad / (torch.sqrt(acc) + f32(eps)))
        else:
            raise ValueError("Could not interpret optimizer identifier: %s" % self.name)

    def step(self, named_vars_grads, touched=None):
        """touched: {key: LongTensor of row ids} -- required in lazy mode."""
        self.t += 1
        for key, (var, grad) in named_vars_grads.items():
            if not self.lazy:
                self.apply(var, grad, key)
                continue
            rows = torch.unique(touched[key])
            full = self.slots.get(key)
            sub_var = var[rows].clone()
            saved = self.slots.get(key)
            # run the dense rule on the touched rows only, with row-sliced slots
            if saved is not None:
                self.slots[key] = tuple(s[rows].clone() for s in saved) if isinstance(saved, tuple) else saved[rows].clone()
            elif self.name == "adam":
                self.slots[key] = (torch.zeros_like(sub_var), torch.zeros_like(sub_var))
                saved = (torch.zeros_like(var), torch.zeros_like(var))
            elif self.name == "adagrad":
                init = float(self.hp.get("initial_accumulator_value", 0.1))
                self.slots[key] = torch.full_like(sub_var, init)
                saved = torch.full_like(var, init)
            self.apply(sub_var, grad[rows], key)
            var[rows] = sub_var
            new = self.slots.get(key)
            if new is not None:
                if isinstance(new, tuple):
                    for s_full, s_new in zip(saved, new):
                        s_full[rows] = s_new
                else:
                    saved[rows] = new
                self.slots[key] = saved


# --------------------------------------------------------------------------
# the step: ScoringBasedEmbeddingModel.call :237-269 + train_step :370-429
# --------------------------------------------------------------------------
class RefStep:
    """One model instance: two fp32 tables + optimizer slots, trained the way
    the reference graph does it (6 gathers per step: s,p,o for the positives
    AND re-gathered s,p,o for every corruption)."""

    def __init__(self, model, K, ent, rel, eta, loss="pairwise", loss_params=None,
                 optimizer="adam", optimizer_params=None, regularizer=None):
        self.model, self.K, self.eta = model, K, eta
        self.ent = torch.as_tensor(np.array(ent, dtype=np.float32)).clone().requires_grad_(True)
        self.rel = torch.as_tensor(np.array(rel, dtype=np.float32)).clone().requires_grad_(True)
        self.max_rel_size = self.rel.shape[0]
        self.loss = loss
        self.loss_params = dict(loss_params or {})
        op = dict(optimizer_params or {})
        self.opt = LegacyOptimizer(optimizer, op.pop("learning_rate", 0.001), **op)
        self.regularizer = regularizer  # None or dict(p=..., lam=...)

    def forward(self, triples, corruptions):
        t = torch.as_tensor(triples, dtype=torch.long)
        e_s, e_p, e_o = self.ent[t[:, 0]], self.rel[t[:, 1]], self.ent[t[:, 2]]  # EmbeddingLookupLayer.py:332-334
        sp = compute_scores(self.model, e_s, e_p, e_o, self.max_rel_size)
        c = torch.as_tensor(corruptions, dtype=torch.long)
        c_s, c_p, c_o = self.ent[c[:, 0]], self.rel[c[:, 1]], self.ent[c[:, 2]]
        sn = compute_scores(self.model, c_s, c_p, c_o, self.max_rel_size)
        return sp, sn

    def loss_and_grads(self, triples, corruptions):
        for v in (self.ent, self.rel):
            v.grad = None
        sp, sn = self.forward(triples, corruptions)
        regs = []
        if self.regularizer:
            regs = [lp_regularizer(self.ent, self.regularizer.get("lam", 1e-5), self.regularizer.get("p", 2)),
                    lp_regularizer(self.rel, self.regularizer.get("lam", 1e-5), self.regularizer.get("p", 2))]
        loss = total_loss(self.loss, sp, sn, self.eta, regs, **self.loss_params)
        loss.backward()  # optimizers.py:166 tape.gradient
        return loss.detach(), sp.detach(), sn.detach(), self.ent.grad, self.rel.grad

    def train_step(self, triples, corruptions):
        loss, sp, sn, g_ent, g_rel = self.loss_and_grads(triples, corruptions)
        with torch.no_grad():  # optimizers.py:168 apply_gradients
            touched = None
            if self.opt.lazy:
                t = torch.as_tensor(triples, dtype=torch.long)
                c = torch.as_tensor(corruptions, dtype=torch.long)
                touched = {"ent": torch.cat([t[:, 0], t[:, 2], c[:, 0], c[:, 2]]), "rel": t[:, 1]}
            self.opt.step({"ent": (self.ent, g_ent), "rel": (self.rel, g_rel)}, touched)
        return float(loss)
