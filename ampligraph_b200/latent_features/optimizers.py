"""Optimizer selection of the facade (mirror of ampligraph/latent_features/optimizers.py).

The reference wraps tf.keras.optimizers.legacy.* (optimizers.py:255-291); here the
update itself is csrc/kge_optim.cu and this wrapper only carries name +
hyper-parameters.  Supported: 'sgd' (optional momentum), 'adam', 'adagrad', 'rmsprop'
(rho, momentum, centered; not centered with momentum), 'adadelta' (rho), 'adamax', 'nadam'
(beta_1, beta_2, epsilon, decay = Keras' schedule_decay) and 'ftrl' (learning_rate_power,
initial_accumulator_value, l1_/l2_/l2_shrinkage_regularization_strength, beta).

get() resolves a name string to one of NAMES, the six kinds built first and their 'lazy_' forms; Nadam and Ftrl are
selected with a Keras optimizer instance (get(tf.keras.optimizers.legacy.Nadam(...)): its get_config() names the kind
and carries its hyper-parameters) or an OptimizerWrapper('nadam' | 'ftrl' | 'lazy_nadam' | 'lazy_ftrl', hyperparams).
"""
KINDS = ("sgd", "adam", "adagrad", "rmsprop", "adadelta", "adamax", "nadam", "ftrl")
# the Keras config keys the facade carries (optimizers.get of a Keras optimizer instance keeps these)
CONFIG_KEYS = ("learning_rate", "beta_1", "beta_2", "epsilon", "momentum", "initial_accumulator_value", "rho", "centered",
               "decay", "schedule_decay", "learning_rate_power", "l1_regularization_strength",
               "l2_regularization_strength", "l2_shrinkage_regularization_strength", "beta")
# extension (not in the reference): 'lazy_<name>' updates only the looked-up rows of both tables, for tables too large
# for the dense rule
SUPPORTED = KINDS + tuple("lazy_" + k for k in KINDS)
# the names get() resolves from a string (see the module docstring)
NAMES = tuple(k for k in SUPPORTED if k.replace("lazy_", "") not in ("nadam", "ftrl"))


class OptimizerWrapper:
    def __init__(self, name="adam", hyperparams=None):
        name = name.lower()
        if name not in SUPPORTED:
            raise ValueError("Could not interpret optimizer identifier: ", name)
        self.name = name
        self.hyperparams = dict(hyperparams or {})
        self.hyperparams.setdefault("learning_rate", 0.001)  # optimizers.py:284
        # adam has beta_1/beta_2 slots (optimizers.py:119-120)
        self.number_hyperparams = 2 if name in ("adam", "lazy_adam") else 1  # Nadam is not an Adam subclass

    def get_hyperparam_count(self):
        return self.number_hyperparams

    def get_config(self):
        return dict(self.hyperparams, name=self.name)


def get(identifier, hyperparams=None):
    """optimizers.get (:255-291): wrapper instance | name of NAMES | object with get_config() (a Keras optimizer
    instance, any of the eight kinds)."""
    if isinstance(identifier, OptimizerWrapper):
        return identifier
    if isinstance(identifier, str):
        if identifier.lower() not in NAMES:
            raise ValueError("Could not interpret optimizer identifier: ", identifier)
        return OptimizerWrapper(identifier, dict(hyperparams or {}))
    cfg = getattr(identifier, "get_config", None)
    if callable(cfg):  # e.g. a Keras optimizer instance: take its config
        c = dict(cfg())
        name = c.pop("name", type(identifier).__name__)
        keep = {k: c[k] for k in CONFIG_KEYS if k in c}
        if str(name).lower() != "nadam":
            keep.pop("decay", None)  # the other kinds' `decay` is Keras' learning-rate time decay (not supported)
        return OptimizerWrapper(str(name), keep)
    raise ValueError("Could not interpret optimizer identifier: ", identifier)


def table_rules(name, hyperparams, regularized):
    """Which tables take the optimizer's IndexedSlices rule, as the reference trains them -> (entities, relations) bools.

    name: an optimizer name of SUPPORTED; hyperparams: its hyper-parameters; regularized: (entities, relations), whether
    each table has a regulariser.  In the reference a table's gradient is the IndexedSlices of tf.nn.embedding_lookup
    (EmbeddingLookupLayer.py:332-339) unless the table has a regulariser or the optimizer is Adagrad, Adadelta or Ftrl (the
    gpu_workaround classes, optimizers.py:50-54,118-121,157-163): those gradients are dense and the dense rule moves every row.
    On IndexedSlices, RMSprop with momentum (ResourceSparseApplyRMSProp) and Adamax update the looked-up rows only, slots
    included.  SGD without momentum, Adam and RMSprop without momentum come to the dense rule's result there: Adam
    decays its slots and moves every row, RMSprop decays ms on every row and a row without a gradient does not move.
    Nadam's IndexedSlices rule (True for Nadam) decays m and v on every row and moves the looked-up rows only
    (KGEEngine.set_optimizer runs it with kge_optimizer_step_decay).
    'lazy_<name>' asks for the looked-up rows on both tables.  SGD with momentum stays dense (DESIGN.md 9)."""
    name = name.lower()
    if name.startswith("lazy_"):
        return True, True
    sparse = name in ("adamax", "nadam") or (name == "rmsprop" and float(dict(hyperparams or {}).get("momentum", 0.0)) != 0.0)
    return tuple(sparse and not bool(r) for r in regularized)
