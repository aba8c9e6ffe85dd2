"""Regulariser selection (mirror of ampligraph/latent_features/regularizers.py + what
`tf.keras.regularizers.get` resolves in EmbeddingLookupLayer.set_regularizer, layers/encoding/EmbeddingLookupLayer.py:131-155).

LP_regularizer = lambda * sum(|x|^p) over the WHOLE table (regularizers.py:14-37); its
loss and dense gradient are fused into the optimizer kernel (csrc/kge_optim.cu).  Keras' 'l1', 'l2' and
'l1_l2' are the same thing with p = 1 / 2 (/ both) and Keras' default factor 0.01.  `compile` accepts one
regulariser for both tables or a list [entities, relations], exactly like the reference.

N3 (extension, not in the reference): the weighted nuclear 3-norm of Lacroix, Usunier and Obozinski (ICML 2018, eq. 6),
lambda * sum of |z_d|^3 over the rows the step's positives use, once per occurrence; |z_d| is the complex modulus for
the two-half layouts.  Its loss and row-sparse gradient come from csrc/kge_reg_n3.cu (DESIGN.md 3.15).

DURA (extension, not in the reference): the duality-induced regulariser of Zhang, Cai and Wang (NeurIPS 2020),
lambda * (alpha (|h|^2 + |t|^2) + beta (|h o r|^2 + |t o conj(r)|^2)) of each of the step's positives, once per
occurrence.  It couples each positive's entity and relation rows, so it is one regulariser of both tables.  With
beta = 0 it is the per-occurrence ("frequency-weighted") squared L2 of the entity rows.  Its loss and row-sparse
gradient come from csrc/kge_reg_dura.cu (DESIGN.md 3.16).
"""
import math


class LPRegularizer:
    __name__ = "LP"

    def __init__(self, regularizer_parameters=None):
        rp = dict(regularizer_parameters or {})
        self.p = int(rp.get("p", 2))
        self.lam = float(rp.get("lambda", 0.00001))
        self.p2 = int(rp.get("p2", 0))        # optional second term (Keras L1L2)
        self.lam2 = float(rp.get("lambda2", 0.0))
        if self.p < 1 or self.p2 < 0:
            raise ValueError("LP regularizer: p must be >= 1")

    def kernel_params(self):
        d = {"p": self.p, "lambda": self.lam}
        if self.p2:
            d.update(p2=self.p2, lambda2=self.lam2)
        return d


def LP_regularizer(regularizer_parameters=None):
    return LPRegularizer(regularizer_parameters)


class N3Regularizer:
    """N3: lambda * sum over the step's positives (s, p, o) of sum_d |z_d|^3 of each of their rows (DESIGN.md 3.15).
    regularizer_parameters: {"lambda": lambda}, default 1e-3 (no precedent here: LP's 1e-5 is a whole-table weight)."""
    __name__ = "N3"

    def __init__(self, regularizer_parameters=None):
        rp = dict(regularizer_parameters or {})
        self.lam = float(rp.get("lambda", 0.001))
        if not self.lam >= 0.0 or self.lam == float("inf"):
            raise ValueError("N3 regularizer: lambda must be finite and >= 0, got %r" % (rp.get("lambda"),))

    def kernel_params(self):
        return {"kind": "N3", "lambda": self.lam}


def N3_regularizer(regularizer_parameters=None):
    return N3Regularizer(regularizer_parameters)


def is_n3(params):
    """Whether a regulariser's kernel_params() (or None) is N3's."""
    return params is not None and params.get("kind") == "N3"


class DURARegularizer:
    """DURA: lambda * sum over the step's positives (h, r, t) of alpha (|h|^2 + |t|^2) + beta (|h o r|^2 + |t o conj(r)|^2)
    (DESIGN.md 3.16).  regularizer_parameters: {"lambda": lambda, "alpha": alpha, "beta": beta}, defaults 1e-3, 1 and 1
    (lambda as N3's: a per-occurrence weight).  Each must be finite and >= 0, and lambda alpha + lambda beta > 0."""
    __name__ = "DURA"

    def __init__(self, regularizer_parameters=None):
        rp = dict(regularizer_parameters or {})
        self.lam, self.alpha, self.beta = (float(rp.get(key, default))
                                           for key, default in (("lambda", 0.001), ("alpha", 1.0), ("beta", 1.0)))
        for key, v in (("lambda", self.lam), ("alpha", self.alpha), ("beta", self.beta)):
            if not (math.isfinite(v) and v >= 0.0):
                raise ValueError("DURA regularizer: %s must be finite and >= 0, got %r" % (key, rp.get(key)))
        if not self.lam * self.alpha + self.lam * self.beta > 0.0:
            raise ValueError("DURA regularizer: lambda * alpha + lambda * beta must be > 0, got lambda %r, alpha %r, "
                             "beta %r" % (self.lam, self.alpha, self.beta))

    def kernel_params(self):
        return {"kind": "DURA", "lambda": self.lam, "alpha": self.alpha, "beta": self.beta}


def DURA_regularizer(regularizer_parameters=None):
    return DURARegularizer(regularizer_parameters)


def is_per_occurrence(params):
    """Whether a regulariser's kernel_params() (or None) penalises the rows each step's positives use, once per occurrence
    (N3, DURA): its gradient lives on the looked-up rows only, like the data term's."""
    return params is not None and params.get("kind") in ("N3", "DURA")


def get(identifier, hyperparams=None):
    """regularizers.get (:40-73) + tf.keras.regularizers.get: 'LP' | 'l3' | 'l1' | 'l2' | 'l1_l2' |
    {'class_name': 'L1'|'L2'|'L1L2', 'config': {...}} | LPRegularizer | None; and 'N3' / 'n3' | N3Regularizer, 'DURA' /
    'dura' | DURARegularizer."""
    hyperparams = dict(hyperparams or {})
    if identifier is None or isinstance(identifier, (LPRegularizer, N3Regularizer, DURARegularizer)):
        return identifier
    if isinstance(identifier, dict):
        cfg = dict(identifier.get("config", {}))
        name = str(identifier.get("class_name", "")).lower()
        if name == "l1":
            return LPRegularizer({"p": 1, "lambda": cfg.get("l1", 0.01)})
        if name == "l2":
            return LPRegularizer({"p": 2, "lambda": cfg.get("l2", 0.01)})
        if name == "l1l2":
            return LPRegularizer({"p": 1, "lambda": cfg.get("l1", 0.0), "p2": 2, "lambda2": cfg.get("l2", 0.0)})
        raise ValueError("Could not interpret regularizer identifier: %r" % (identifier,))
    if isinstance(identifier, str):
        key = identifier.lower()
        if identifier == "l3":
            hyperparams["p"] = 3
            return LPRegularizer(hyperparams)
        if identifier == "LP":
            return LPRegularizer(hyperparams)
        if key == "n3":
            return N3Regularizer(hyperparams)
        if key == "dura":
            return DURARegularizer(hyperparams)
        if key == "l2":  # Keras 'l2': 0.01 * sum(x^2)
            return LPRegularizer({"p": 2, "lambda": hyperparams.get("lambda", 0.01)})
        if key == "l1":
            return LPRegularizer({"p": 1, "lambda": hyperparams.get("lambda", 0.01)})
        if key == "l1_l2":
            return LPRegularizer({"p": 1, "lambda": hyperparams.get("l1", 0.01), "p2": 2, "lambda2": hyperparams.get("l2", 0.01)})
    raise ValueError("Could not interpret regularizer identifier: %r" % (identifier,))


def get_pair(identifier, hyperparams=None):
    """One regulariser for both tables, or a list of two [entities, relations] (EmbeddingLookupLayer.py:145-155)."""
    if isinstance(identifier, (list, tuple)):
        assert len(identifier) == 2, "Incorrect length for regularizer. Expected 2, got {}".format(len(identifier))
        return [get(identifier[0], hyperparams), get(identifier[1], hyperparams)]
    r = get(identifier, hyperparams)
    return [r, r]
