"""Optimizer selection of the facade (mirror of ampligraph/latent_features/optimizers.py).

The reference wraps tf.keras.optimizers.legacy.* (optimizers.py:255-291); here the
update itself is csrc/kge_optim.cu and this wrapper only carries name +
hyper-parameters.  Supported: 'sgd' (optional momentum), 'adam', 'adagrad', 'rmsprop'
(rho, momentum, centered; not centered with momentum), 'adadelta' (rho), 'adamax'.
"""
KINDS = ("sgd", "adam", "adagrad", "rmsprop", "adadelta", "adamax")
# extension (not in the reference): 'lazy_<name>' updates only the looked-up rows of both tables, for tables too large
# for the dense rule
SUPPORTED = KINDS + tuple("lazy_" + k for k in KINDS)


class OptimizerWrapper:
    def __init__(self, name="adam", hyperparams=None):
        name = name.lower()
        if name not in SUPPORTED:
            raise ValueError("Could not interpret optimizer identifier: ", name)
        self.name = name
        self.hyperparams = dict(hyperparams or {})
        self.hyperparams.setdefault("learning_rate", 0.001)  # optimizers.py:284
        # adam has beta_1/beta_2 slots (optimizers.py:119-120)
        self.number_hyperparams = 2 if name.endswith("adam") else 1

    def get_hyperparam_count(self):
        return self.number_hyperparams

    def get_config(self):
        return dict(self.hyperparams, name=self.name)


def get(identifier, hyperparams=None):
    """optimizers.get (:255-291): wrapper instance | name | object with get_config()."""
    if isinstance(identifier, OptimizerWrapper):
        return identifier
    if isinstance(identifier, str):
        return OptimizerWrapper(identifier, dict(hyperparams or {}))
    cfg = getattr(identifier, "get_config", None)
    if callable(cfg):  # e.g. a Keras optimizer instance: take its config
        c = dict(cfg())
        name = c.pop("name", type(identifier).__name__)
        keep = {k: c[k] for k in ("learning_rate", "beta_1", "beta_2", "epsilon", "momentum",
                                  "initial_accumulator_value", "rho", "centered") if k in c}
        return OptimizerWrapper(str(name), keep)
    raise ValueError("Could not interpret optimizer identifier: ", identifier)


def table_rules(name, hyperparams, regularized):
    """Which tables take the looked-up-rows rule, as the reference trains them -> (entities, relations) bools.

    name: an optimizer name of SUPPORTED; hyperparams: its hyper-parameters; regularized: (entities, relations), whether
    each table has a regulariser.  In the reference a table's gradient is the IndexedSlices of tf.nn.embedding_lookup
    (EmbeddingLookupLayer.py:332-339) unless the table has a regulariser or the optimizer is Adagrad or Adadelta (the
    gpu_workaround classes, optimizers.py:118-121,157-163): those gradients are dense and the dense rule moves every row.
    On IndexedSlices, RMSprop with momentum (ResourceSparseApplyRMSProp) and Adamax update the looked-up rows only, slots
    included.  SGD without momentum, Adam and RMSprop without momentum come to the dense rule's result there: Adam
    decays its slots and moves every row, RMSprop decays ms on every row and a row without a gradient does not move.
    'lazy_<name>' asks for the looked-up rows on both tables.  SGD with momentum stays dense (DESIGN.md 9)."""
    name = name.lower()
    if name.startswith("lazy_"):
        return True, True
    sparse = name == "adamax" or (name == "rmsprop" and float(dict(hyperparams or {}).get("momentum", 0.0)) != 0.0)
    return tuple(sparse and not bool(r) for r in regularized)
