"""ScoringBasedEmbeddingModel facade: the reference's fit / predict / evaluate surface
(ampligraph/latent_features/models/ScoringBasedEmbeddingModel.py) re-hosted on
KGEEngine.  Only the loops and the host-side data plumbing live here; every number is
produced by libkge_b200.so.
"""
import math
import numbers
import pickle

import numpy as np
import torch

from .. import _lib
from ..datasets import (NEGATIVE_SAMPLERS, DataIndexer, FilterIndex, as_triple_array, k_vs_all_queries, k_vs_all_steps,
                        negative_sampler_tables, nscaching_tables, reciprocal_triples)
from ..engine import KGEEngine, NegativeSamplerTables, NSCache
from ..evaluation import hits_at_n_score, mr_score, mrr_score, train_test_split_no_unseen
from . import initializers, loss_functions, optimizers, regularizers
from .layers.scoring import SCORING_LAYER_REGISTRY

NEGATIVE_FILTER_ATTEMPTS = 10  # draws of a corruption's entity under fit(filter_negatives=True) (DESIGN.md 3.18)
FIT_NEGATIVE_SAMPLERS = NEGATIVE_SAMPLERS + ("nscaching",)
NSCACHING_PARAMS = {"cache_size": 50, "random_size": 50}  # N1, N2: the paper's defaults (DESIGN.md 3.20)
NSCACHING_MAX_CANDIDATES = 512  # N1 + N2: the refresh kernel's candidates per row


class History:
    """Stand-in for the Keras History callback object returned by fit()."""

    def __init__(self):
        self.history = {}
        self.epoch = []

    def _log(self, epoch, logs):
        self.epoch.append(epoch)
        for k, v in logs.items():
            self.history.setdefault(k, []).append(v)


class EarlyStopping:
    """tf.keras.callbacks.EarlyStopping (Keras 2.15) used with fit(validation_data=...): stop when `monitor`
    (e.g. 'val_mrr') has not improved by more than `min_delta` for `patience` epochs that report it.

    Keras's rule: epochs without the monitored value are skipped; every other epoch counts one towards `wait`, and an
    improvement sets `best`, resets `wait` to 0 and, with restore_best_weights, snapshots the tables (the first monitored
    epoch always does).  Training stops when wait >= patience at an epoch other than the first, and the tables are then
    set back to the snapshot.  The snapshot is the entity and relation tables only, as Keras's get_weights: optimizer
    slots and the step count keep their values.  fit() calls on_train_begin, which starts each fit afresh, so one
    instance can serve several fits.  mode='auto' means 'min' for a monitor containing 'loss' or ending in 'mr', else
    'max' (Keras's own 'auto' would minimise MRR and hits).  stopped_epoch is None when training was not stopped."""

    def __init__(self, monitor="val_mrr", min_delta=0.0, patience=0, mode="auto", restore_best_weights=False, verbose=0):
        self.monitor, self.min_delta, self.patience = monitor, abs(min_delta), patience
        self.restore_best_weights, self.verbose = restore_best_weights, verbose
        if mode == "auto":
            mode = "min" if ("loss" in monitor or monitor.endswith("mr")) else "max"
        self.sign = 1.0 if mode == "max" else -1.0
        self.model = None
        self.on_train_begin()

    def on_train_begin(self, logs=None):
        self.best, self.best_epoch, self.wait, self.stopped_epoch, self.best_weights = -self.sign * np.inf, 0, 0, None, None

    def on_epoch_end(self, epoch, logs):
        if self.monitor not in logs:
            return
        current = float(logs[self.monitor])
        if self.restore_best_weights and self.best_weights is None:
            self.best_weights = self.model._snapshot_tables()
        self.wait += 1
        if self.sign * (current - self.best) - self.min_delta > 0:
            self.best, self.best_epoch, self.wait = current, epoch, 0
            if self.restore_best_weights:
                self.best_weights = self.model._snapshot_tables()
            return
        if self.wait >= self.patience and epoch > 0 and self.model is not None:
            self.stopped_epoch = epoch
            self.model.stop_training = True
            if self.restore_best_weights:
                if self.verbose > 0:
                    print("Restoring model weights from the end of the best epoch: %d." % (self.best_epoch + 1))
                self.model._restore_tables(self.best_weights)


class ScoringBasedEmbeddingModel:
    """Same constructor as the reference (ScoringBasedEmbeddingModel.py:100-171).

    reciprocal_relations (extension; DESIGN.md 3.17): True gives each of the max_rel_size (R) relations p a second,
    independently learned row p^-1 (row p + R of the relation table, which has 2R rows).  Every training triple
    (s, p, o) then also trains its inverse (o, p^-1, s), and a subject query (?, p, o) is answered as the object query
    (o, p^-1, ?) (Lacroix et al., ICML 2018).  predict scores the forward triple f(s, p, o), and relation ranking and
    top-n consider the forward relations only.  It needs DistMult, ComplEx or HolE trained with fit(one_vs_all=...) or
    fit(k_vs_all=...) on one GPU, without the relation-prediction term: every other training path is refused."""

    def __init__(self, eta, k, scoring_type="DistMult", seed=0, max_ent_size=None, max_rel_size=None,
                 reciprocal_relations=False):
        if scoring_type not in SCORING_LAYER_REGISTRY:
            raise KeyError(scoring_type)  # the reference indexes the registry directly (:146)
        if reciprocal_relations and scoring_type in ("TransE", "RotatE"):
            raise NotImplementedError("reciprocal relations need 1vsAll or KvsAll training, which is implemented for "
                                      "DistMult, ComplEx and HolE, not for %s" % scoring_type)
        self.reciprocal_relations = bool(reciprocal_relations)
        self.eta, self.k, self.scoring_type, self.seed = int(eta), int(k), scoring_type, seed
        self.max_ent_size, self.max_rel_size = max_ent_size, max_rel_size
        self.scoring_layer = SCORING_LAYER_REGISTRY[scoring_type](k)
        if self.scoring_layer.kernel_id is None:
            raise NotImplementedError("scoring_type %r is the reference's random baseline: it is registered for parity of "
                                      "the registry only and has no CUDA kernel" % scoring_type)
        self.internal_k = self.scoring_layer.internal_k
        self.data_indexer = True
        self.is_fitted = False
        self.is_calibrated = False
        self.is_partitioned_training = False
        self._is_compiled = False
        self.engine = None
        self.device = 0
        self._loss_sum, self._loss_cnt = 0.0, 0  # never-reset running Mean metric (loss_functions.py:101,:224)
        self._initial_tables = None
        self._step = 0
        # set True (under torchrun, after torch.distributed.init_process_group) to train data-parallel over
        # all ranks -- every global batch is split across ranks -- and to rank against row shards
        self.distributed = False
        self._dp = None
        self.use_focusE = False
        self.negative_filter_misses = 0  # known corruptions the last fit(filter_negatives=True) trained on

    # ------------------------------------------------------------------ compile
    def compile(self, optimizer="adam", loss=None, entity_relation_initializer="glorot_uniform",
                entity_relation_regularizer=None, **kwargs):
        """compile (:1145-1318).  entity_relation_initializer: anything tf.keras.initializers.get takes in the reference
        (a name such as 'glorot_uniform' / 'random_normal' / 'he_uniform', a {'class_name', 'config'} dict, an
        initializers.Initializer instance), an ndarray, a callable(shape)->ndarray, or a list of two of those
        [entities, relations] (EmbeddingLookupLayer.py:105-129).  entity_relation_regularizer: None | 'LP' | 'l3' |
        'l1' | 'l2' | 'l1_l2' | regularizers.LPRegularizer, or a list of two [entities, relations] (:131-155).
        'N3' | regularizers.N3Regularizer (extension; DESIGN.md 3.15): lambda * sum_d |z_d|^3 of the rows each step's
        positives use, once per occurrence (|z_d| the complex modulus for ComplEx, HolE and RotatE), default lambda
        1e-3, e.g. ['N3', None] for the entities only.  It is not defined for RotatE's relation phases, and not with
        k_vs_all training or on several GPUs.
        'DURA' | regularizers.DURARegularizer (extension; DESIGN.md 3.16): lambda * (alpha (|h|^2 + |t|^2) + beta
        (|h o r|^2 + |t o conj(r)|^2)) of each step's positives, once per occurrence (|.| the complex modulus for ComplEx
        and HolE), defaults lambda 1e-3, alpha = beta = 1.  It couples each positive's entity and relation rows, so it is
        only valid as the single regularizer of both tables, not in a list.  It needs DistMult, ComplEx or HolE, and is
        not supported with k_vs_all training or on several GPUs.
        With reciprocal relations the relation initializer covers the 2R rows of the relation table, forward rows then
        inverse rows: a callable is called with the shape (2R, internal_k), an ndarray must have that shape, and the
        device-side Glorot draw's limit sqrt(6 / (fan_in + fan_out)) counts the 2R rows."""
        self.optimizer = optimizers.get(optimizer)
        self.compiled_loss = loss_functions.get(loss)
        init = entity_relation_initializer
        if isinstance(init, (list, tuple)):
            assert len(init) == 2, "Incorrect length for initializer. Assumed 2 got {}".format(len(init))
            self._initializer = [initializers.get(init[0]), initializers.get(init[1])]
        else:
            self._initializer = [initializers.get(init), initializers.get(init)]
        if self.scoring_type == "RotatE":  # :1312-1315
            r = self._initializer[1]
            assert isinstance(r, initializers.Initializer) and r.name == "glorot_uniform", \
                "The relation initializer provided to a RotatE model must be glorot_uniform!"
        self._regularizer = regularizers.get_pair(entity_relation_regularizer)
        if isinstance(entity_relation_regularizer, (list, tuple)) and self._uses_dura():
            raise ValueError("the DURA regularizer couples each positive's entity and relation rows, so it cannot be "
                             "given per table: pass it as the single entity_relation_regularizer, not in a list")
        if self.scoring_type in ("TransE", "RotatE") and self._uses_dura():
            raise NotImplementedError("the DURA regularizer is defined for the tensor-factorisation models (DistMult, "
                                      "ComplEx, HolE), not for %s" % self.scoring_type)
        if self.scoring_type == "RotatE" and isinstance(self._regularizer[1], regularizers.N3Regularizer):
            raise NotImplementedError("the N3 regularizer is not defined for RotatE's relation table (its rows are "
                                      "phases, not embeddings): use ['N3', None]")
        self._loss_sum, self._loss_cnt = 0.0, 0
        self._is_compiled = True
        self.engine = None  # tables are (re)built lazily on the first fit, like EmbeddingLookupLayer.build

    def _assert_compile_was_called(self):
        if not self._is_compiled:
            raise RuntimeError("You must compile your model before training/testing. Use `model.compile(optimizer, loss)`.")

    def is_fit(self):
        return self.is_fitted

    # ------------------------------------------------------------------ engine
    def _build_engine(self):
        name, lp = self.compiled_loss.kernel_params()
        reg = [r.kernel_params() if r is not None else None for r in self._regularizer]
        if self.scoring_type == "RotatE":
            self.scoring_layer.max_rel_size = self.max_rel_size  # :338
        # the reference's per-table rule: which tables its optimizer updates on the looked-up rows only
        # a per-occurrence regulariser's (N3, DURA) gradient lives on the looked-up rows only, like the data term's: it
        # does not make a table's gradient dense
        lazy = optimizers.table_rules(self.optimizer.name, self.optimizer.hyperparams,
                                      [r is not None and not regularizers.is_per_occurrence(r) for r in reg])

        rel_rows = self._rel_rows()

        def make_engine(alloc=None):
            return KGEEngine(self.scoring_type, self.k, self.eta, self.max_ent_size, rel_rows,
                             loss=name or "pairwise", loss_params=lp, optimizer=self.optimizer.name,
                             optimizer_params=self.optimizer.hyperparams, regularizer=reg, device=self.device,
                             table_alloc=alloc, lazy_tables=lazy)
        if self._world() > 1:
            from ..parallel import DataParallelTrainer
            self._dp = DataParallelTrainer(make_engine)
            self.engine = self._dp.eng
        else:
            self.engine = make_engine()
        dense = [None, None]
        for n, (init, rows, which) in enumerate(zip(self._initializer, (self.max_ent_size, rel_rows), ("ent", "rel"))):
            if isinstance(init, initializers.Initializer):  # drawn on the device (Philox), no host table
                seed = init.seed if getattr(init, "seed", None) is not None else self.seed
                if init.name == "glorot_uniform":
                    self.engine.init_glorot_uniform(seed, only=which)
                else:
                    kind, a, b = init.spec(rows, self.internal_k)
                    self.engine.init_table(which, kind, a, b, seed)
            elif callable(init):
                dense[n] = np.asarray(init((rows, self.internal_k)), dtype=np.float32)
            else:
                dense[n] = np.asarray(init, dtype=np.float32)
                if which == "rel" and self.reciprocal_relations and dense[n].shape != (rows, self.internal_k):
                    raise ValueError("with reciprocal relations the relation initializer needs shape %s (2R rows: the "
                                     "%d forward relations, then their inverses), got shape %s"
                                     % ((rows, self.internal_k), self.max_rel_size, dense[n].shape))
        self.engine.set_embeddings(dense[0], dense[1])
        self._step = 0

    def _rel_rows(self):
        """Rows of the relation table: R, or 2R with reciprocal relations (row p + R is the inverse of relation p)."""
        return 2 * self.max_rel_size if self.reciprocal_relations else self.max_rel_size

    def _world(self):
        import torch.distributed as dist
        return dist.get_world_size() if (self.distributed and dist.is_available() and dist.is_initialized()) else 1

    def _rank(self):
        import torch.distributed as dist
        return dist.get_rank() if self._world() > 1 else 0

    def _to_dev(self, a, dtype):
        """host array -> device tensor.  Pageable source, synchronous copy: these are the small per-chunk id / filter
        arrays of evaluate and the one-off upload of fit; pinning a fresh buffer per call (round 1) cost more than the
        copy.  The per-step training path stages batches through ONE persistent pinned ring (train_on_batches)."""
        return torch.as_tensor(np.ascontiguousarray(a, dtype=dtype)).to(self.engine.device)

    # ------------------------------------------------------------------ indexing
    def _index(self, x, fit=False):
        x = as_triple_array(x)
        if self.data_indexer is False:  # use_indexer=False: data is already int ids
            t = np.ascontiguousarray(x[:, :3], dtype=np.int32)
            if self.reciprocal_relations and self.max_rel_size is not None and (t[:, 1] >= self.max_rel_size).any():
                raise ValueError("relation ids must be below max_rel_size = %d: with reciprocal relations the rows "
                                 "from %d on are the inverse relations" % (self.max_rel_size, self.max_rel_size))
            return t
        if fit and not isinstance(self.data_indexer, DataIndexer):
            self.data_indexer = DataIndexer(x[:, :3])
        return self.data_indexer.get_indexes(x[:, :3], "t", "raw2ind")

    def get_indexes(self, X, type_of="t", order="raw2ind"):
        return self.data_indexer.get_indexes(X, type_of, order)

    def get_count(self, concept_type="e"):
        if concept_type == "e":
            return self.data_indexer.get_entities_count()
        if concept_type == "r":
            return self.data_indexer.get_relations_count()
        raise ValueError("Invalid Concept Type (expected 'e' or 'r')")

    # ------------------------------------------------------------------ fit
    def fit(self, x=None, batch_size=1000, epochs=100, verbose=True, callbacks=None, validation_split=0.0,
            validation_data=None, shuffle=True, initial_epoch=0, validation_batch_size=10,
            validation_corrupt_side="s,o", validation_freq=10, validation_burn_in=0, validation_filter=False,
            validation_entities_subset=None, partitioning_k=1, focusE=False, focusE_params={}, one_vs_all=None,
            k_vs_all=None, label_smoothing=0.0, relation_prediction_weight=0.0, negative_sampler="uniform",
            filter_negatives=False, entity_dropout=0.0, relation_dropout=0.0, negative_sampler_params=None,
            shared_negatives=0):
        """fit (:544-883).  `shuffle` is accepted and ignored exactly like the reference
        (batches are the sequential slices of graph_data_loader.py:495-500).  validation_split: carve the validation
        set out of x with train_test_split_no_unseen(x, test_size=validation_split, seed=self.seed), as the reference
        does (:719-727).  The filter of the validations (validation_filter) is indexed once per fit, not per validation.

        one_vs_all (extension): None trains against eta sampled corruptions per positive.  's,o', 'o' or 's' trains
        1vsAll instead (Ruffinelli et al., ICLR 2020): every step scores each positive against every entity on the
        given sides, with the multiclass NLL over all of them (the setting of the reference's multiclass_nll
        docstring, loss_functions.py:580-590; DESIGN.md 3.12).  eta and the corruption seed are then unused.  It needs
        DistMult, ComplEx or HolE and the compiled loss 'multiclass_nll' (either reduction), on one GPU without
        focusE.

        k_vs_all (extension): 's,o', 'o' or 's' trains KvsAll instead (Ruffinelli et al., ICLR 2020; DESIGN.md 3.13):
        every distinct (s, p) of x (side 'o') or (p, o) (side 's') is one training row, scored against every entity,
        with target 1 for its known objects (subjects) in x and 0 for the rest, under the compiled loss 'nll' (binary
        cross-entropy on each (query, entity) pair; reduction 'mean' averages over the n_ent entities).  Queries keep
        the order of their first appearance in x.  With both sides an epoch has ceil((n_o + n_s) / batch_size)
        steps, each taking its share of both sides' queries; one side is cut into slices of batch_size queries.
        label_smoothing eps in [0, 1) sets the targets to (1 - eps) y + eps / n_ent (PyKEEN's convention).  eta and
        the corruption seed are then unused.  It needs DistMult, ComplEx or HolE, on one GPU without focusE, and
        cannot be combined with one_vs_all.

        relation_prediction_weight (extension): lambda >= 0.  With one_vs_all and lambda > 0, every step adds
        lambda * L_p to the 1vsAll loss, L = L_s + L_o + lambda * L_p (Chen et al., "Relation Prediction as an Auxiliary
        Training Objective for Improving Multi-Relational Graph Representations", AKBC 2021; DESIGN.md 3.14): L_p is
        the multiclass NLL of each positive's relation against every relation, scored as f(s, r, o), under the same
        reduction.  The logged loss includes the term.  It needs one_vs_all, at least two relations, and cannot be
        combined with k_vs_all.  0.0 (the default) leaves training unchanged.

        With the N3 or DURA regulariser (compile(entity_relation_regularizer='N3' or 'DURA')), every step adds its
        term of the batch's positives (once per step, also with one_vs_all and relation_prediction_weight; DESIGN.md
        3.15, 3.16) and the logged loss includes it.  Neither can be combined with k_vs_all, whose steps have queries
        rather than triples, and both are single-GPU only.

        With reciprocal_relations (constructor; DESIGN.md 3.17) only one_vs_all and k_vs_all train.  one_vs_all: each
        positive (s, p, o) gives the side-o row (s, p, o) for side 'o' and the side-o row (o, p^-1, s) for side 's', and
        a step is one side-o 1vsAll call over the batch's forward rows, then its inverse rows; the logged loss sums
        both, and N3 / DURA regularise every row the step trained.  k_vs_all: each side-s query (p, o) with labels {s}
        becomes the side-o query (o, p^-1) with the same labels; the epoch's steps and label_smoothing are unchanged.

        negative_sampler, filter_negatives (extension; DESIGN.md 3.18): how sampled training draws its corruptions.
        'uniform' (default) replaces the subject or the object on a fair coin, by any entity.  'bernoulli' replaces the
        subject of relation p with probability tph / (tph + hpt) (Wang et al., AAAI 2014), by any entity.
        'pseudo_typed' keeps the fair coin and draws the replacement from the entities seen in that slot of p in x
        (PyKEEN's PseudoTypedNegativeSampler).  filter_negatives=True draws a corruption that is a triple of x again,
        up to NEGATIVE_FILTER_ATTEMPTS draws; those still known after the last are trained on and counted in
        self.negative_filter_misses (read once per epoch).  The tables are built once per fit from x.  They apply to
        every single-GPU sampled step of fit (the fused step, user losses, focusE), not to one_vs_all or k_vs_all;
        train_on_batch and train_on_batches stay uniform.  'uniform' without the filter is the path fit always took.

        negative_sampler='nscaching' (extension; DESIGN.md 3.20; Zhang et al., ICDE 2019) keeps a cache of
        high-scoring entities for every (s, p) and every (p, o) of x and draws each corruption uniformly from the cache
        of its positive's query, the side on a fair coin.  Every step first refreshes the caches of its batch's queries:
        the cached entities plus random_size uniform ones, with duplicates (and, with filter_negatives=True, triples of
        x) dropped, are sampled down to cache_size without replacement with probability proportional to exp(score) of
        the current embeddings.  negative_sampler_params={"cache_size": N1, "random_size": N2} (ints >= 1,
        N1 + N2 <= 512; default 50 and 50, the paper's) is accepted with 'nscaching' only.  The caches start empty at
        every fit and persist across its epochs.  A corruption of a cache the filter left empty is drawn uniformly and
        counted in self.negative_filter_misses.

        entity_dropout, relation_dropout (extension; DESIGN.md 3.19): p in [0, 1), inverted dropout on the entity and
        relation embedding elements every training score of the fit reads (LibKGE's lookup-embedder dropout, tuned by
        Ruffinelli et al., ICLR 2020): each kept element is scaled by 1 / (1 - p), each dropped one is 0.  A step's
        candidate rows share one mask per side; each query row of the batch draws its own.  The masks come from the
        model's seed and the step.  They apply to one_vs_all and k_vs_all training only (with reciprocal relations,
        relation_prediction_weight, N3, DURA, label smoothing and either reduction); the regularisers, the optimizer,
        validation, evaluate, predict and every later call read the raw embeddings.  The logged loss is that of the
        dropped-out scores.  0.0 (the default) leaves training unchanged.

        shared_negatives (extension; DESIGN.md 3.21; PyTorch-BigGraph, DGL-KE): an int C >= 1 cuts every batch into
        chunks of C consecutive positives (the last may be shorter) and corrupts all positives of a chunk against one
        set of eta candidate entities drawn from (seed, step), each corruption on the side the per-positive sampler
        picks ('uniform' or 'bernoulli').  The GPU step reads a candidate row once per slice of 16 positives of a
        chunk instead of once per positive, whatever C is: C > 16 changes which negatives are drawn, not the cost.
        Measured on an H100 at eta = 256 (DESIGN.md 5), the step is faster than the per-positive one for RotatE and
        TransE at k = 1,000 (1.25x, 1.14x) and slower for ComplEx k = 200 on an FB15k-237-sized table (0.57x), whose
        per-positive step reads its rows from L2; it is not a general speed-up.  Every built-in loss,
        both reductions, N3 / DURA / LP regularisers and every optimizer apply as in the fused step; with C = 1 the
        corruptions are those of the default draw.  It is refused with one_vs_all or k_vs_all, with 'pseudo_typed',
        'nscaching' or filter_negatives=True (ValueError: they pick entities per positive), and with a user loss,
        focusE or several GPUs (NotImplementedError).  0 (the default) trains as before."""
        self._assert_compile_was_called()
        self._check_dropout(entity_dropout, relation_dropout, one_vs_all, k_vs_all)
        if self.reciprocal_relations:
            self._check_reciprocal("fit", one_vs_all, k_vs_all, focusE, relation_prediction_weight)
        sampled_option = self._check_negative_sampler(negative_sampler, filter_negatives, one_vs_all, k_vs_all,
                                                      negative_sampler_params)
        self._check_per_occurrence(k_vs_all)
        if k_vs_all is not None or label_smoothing != 0.0:
            self._check_k_vs_all(k_vs_all, label_smoothing, one_vs_all, focusE)
        if one_vs_all is not None:
            self._check_one_vs_all(one_vs_all, focusE)
        self._check_relation_prediction(relation_prediction_weight, one_vs_all, k_vs_all)
        self._check_shared_negatives(shared_negatives, one_vs_all, k_vs_all, negative_sampler, filter_negatives, focusE)
        if validation_split:
            assert isinstance(x, np.ndarray), "Validation split supported for numpy arrays only!"
            x, validation_data = train_test_split_no_unseen(x, test_size=validation_split, seed=self.seed,
                                                            allow_duplication=False)
        if partitioning_k != 1:
            raise NotImplementedError("bucket partitioning is replaced by HBM-resident tables (DESIGN.md)")
        x = as_triple_array(x)
        # FocusE (:342-368, :396-406, :468-543): numeric edge values in columns 3.. re-weight the scores
        self.use_focusE = bool(focusE) and x.shape[1] > 3
        if x.shape[1] > 3 and not focusE:
            print("Data shape is {}: not only triples were given, but focusE is not active!".format(x.shape[1]))
        if self.use_focusE:
            assert isinstance(focusE_params, dict), "focusE parameters need to be in a dict!"
            from .torch_losses import focuse_non_linearity
            self._focuse_nl = focuse_non_linearity(focusE_params.get("non_linearity", "linear"))
            self._focuse_stop = focusE_params.get("stop_epoch", 251)
            assert self._focuse_stop >= 0, "Invalid value for focusE stop_epoch: expected a value >=0 but got {}".format(self._focuse_stop)
            self._focuse_sw = focusE_params.get("structural_wt", 0.001)
            assert 0 <= self._focuse_sw <= 1, "Invalid focusE 'structural_wt' passed! It has to belong to [0,1]."
        triples = self._index(x, fit=True)
        if self.data_indexer is not False:
            self.max_ent_size = self.data_indexer.get_entities_count()
            self.max_rel_size = self.data_indexer.get_relations_count()
        elif self.max_ent_size is None or self.max_rel_size is None:
            self.max_ent_size = int(max(triples[:, 0].max(), triples[:, 2].max())) + 1
            self.max_rel_size = int(triples[:, 1].max()) + 1
        if relation_prediction_weight > 0 and self.max_rel_size < 2:
            raise ValueError("relation_prediction_weight needs at least two relations, got %d" % self.max_rel_size)
        if self.engine is None:
            self._build_engine()
        eng = self.engine
        dropout = (float(entity_dropout), float(relation_dropout))
        if any(dropout):  # only the all-candidate steps read it; validation ranks the raw embeddings
            eng.set_embedding_dropout(*dropout, seed=self.seed)
        try:
            return self._fit_loop(x, triples, batch_size, epochs, verbose, callbacks, validation_data, initial_epoch,
                                  validation_batch_size, validation_corrupt_side, validation_freq, validation_burn_in,
                                  validation_filter, validation_entities_subset, one_vs_all, k_vs_all, label_smoothing,
                                  relation_prediction_weight, negative_sampler, filter_negatives, sampled_option,
                                  negative_sampler_params, shared_negatives)
        finally:
            if any(dropout):
                eng.set_embedding_dropout(0.0, 0.0)

    def _fit_loop(self, x, triples, batch_size, epochs, verbose, callbacks, validation_data, initial_epoch,
                  validation_batch_size, validation_corrupt_side, validation_freq, validation_burn_in,
                  validation_filter, validation_entities_subset, one_vs_all, k_vs_all, label_smoothing,
                  relation_prediction_weight, negative_sampler, filter_negatives, sampled_option,
                  negative_sampler_params=None, shared_negatives=0):
        """fit's training loop, on the engine fit has built (with fit's embedding dropout set on it)."""
        eng = self.engine
        eng.set_hot_entities(triples=triples)  # the most frequent entities of the training set: their gradient rows are summed per warp
        data = self._to_dev(triples, np.int32)  # uploaded once; batches are device-side slices
        n = data.shape[0]
        ova_rows, ova_sides = None, one_vs_all
        if self.reciprocal_relations and one_vs_all is not None:
            # each batch's forward and inverse rows, adjacent and uploaded once: a step is one side-o call over a slice
            ova_rows = self._to_dev(reciprocal_triples(triples, self.max_rel_size, one_vs_all, batch_size), np.int32)
            ova_sides = "o"
        m = len(one_vs_all.split(",")) if ova_rows is not None else 1
        weights = None
        if self.use_focusE:
            if len(triples) != len(x):
                raise ValueError("focusE needs every input triple to be indexable")
            weights = self._to_dev(np.asarray(x[:, 3:], dtype=np.float32), np.float32)
        batch_size = int(batch_size)
        history = History()
        self.stop_training = False
        user_loss = isinstance(self.compiled_loss, loss_functions.LossFunctionWrapper)
        world, rank = self._world(), self._rank()
        if world > 1 and (user_loss or self.use_focusE):
            raise NotImplementedError("user-callable losses / focusE are single-GPU only")
        val_findex = None  # the FilterIndex of validation_filter, built at the first validation and kept for the others
        for cb in (callbacks or []):  # Keras's set_model + on_train_begin: a callback instance may serve several fits
            try:
                cb.model = self
            except Exception:
                pass
            if hasattr(cb, "on_train_begin"):
                cb.on_train_begin({})
        kva = kva_steps = None
        if k_vs_all is not None:  # each side's queries, label offsets and label ids, uploaded once; steps slice them
            findex = FilterIndex(triples, self.max_ent_size)
            kva = {}
            for side in k_vs_all.split(","):
                q, off, ids = k_vs_all_queries(findex, triples, side)
                if self.reciprocal_relations and side == "s":  # (p, o) with labels {s} -> the side-o query (o, p^-1)
                    q = reciprocal_triples(q, self.max_rel_size, "s")
                kva[side] = tuple(self._to_dev(a, a.dtype) for a in (q, off, ids))
            count = lambda side: kva[side][0].shape[0] if side in kva else 0
            kva_steps = k_vs_all_steps(count("o"), count("s"), batch_size)
        sampler = None
        if negative_sampler == "nscaching":
            params = dict(NSCACHING_PARAMS, **(negative_sampler_params or {}))
            sampler = NSCache(nscaching_tables(triples, self.max_ent_size, self.max_rel_size, batch_size, filter_negatives),
                              params["cache_size"], params["random_size"], eng.device)
            eng.read_negative_misses()  # start this fit's count at 0
        elif sampled_option:
            sampler = NegativeSamplerTables(
                negative_sampler_tables(triples, self.max_ent_size, self.max_rel_size, negative_sampler, filter_negatives),
                NEGATIVE_FILTER_ATTEMPTS, eng.device)
            eng.read_negative_misses()  # start this fit's count at 0
        self.negative_filter_misses = 0
        for epoch in range(initial_epoch, epochs):
            if self.use_focusE and self._focuse_stop > 0:  # linear decay of the structural weight (:536-543)
                self._focuse_sw = max(1 - epoch / self._focuse_stop, 0.001)
            for start in (kva_steps if kva is not None else range(0, n, batch_size)):
                batch = data[start:start + batch_size] if kva is None else None
                if kva is not None:  # start: this step's query ranges of sides o and s
                    self._k_vs_all_step(kva, start, label_smoothing)
                elif one_vs_all is not None:
                    if ova_rows is not None:
                        batch = ova_rows[m * start:m * (start + batch_size)]
                    eng.one_vs_all_backward(batch, ova_sides, step=self._step)
                    if relation_prediction_weight > 0:
                        eng.one_vs_all_relation_backward(batch, relation_prediction_weight, step=self._step)
                    self._per_occurrence_backward(batch)
                    eng.apply_gradients()
                elif shared_negatives:
                    eng.shared_negatives_backward(batch, shared_negatives, seed=self.seed, step=self._step,
                                                  sampler=sampler)
                    self._per_occurrence_backward(batch)
                    eng.apply_gradients()
                elif self.use_focusE:
                    self._two_phase_step(batch, weights[start:start + batch_size], sampler, start)
                else:
                    if world > 1:  # this rank's slice of the global batch; the step is the global-batch step
                        from ..parallel import row_shard
                        lo, hi = row_shard(batch.shape[0], world, rank)
                        batch = batch[lo:hi]
                    self._sampled_step(batch, sampler, start)
                self._step += 1
                self._loss_cnt += 1
            # per-batch losses accumulate on the device; one read-back per epoch (the logged value is
            # the reference's never-reset running mean of per-batch SUM losses)
            if world > 1:
                self._dp.reduce_loss_()
            self._loss_sum += eng.read_loss()
            if sampler is not None:  # after read_loss's synchronisation: no step waits for it
                self.negative_filter_misses += eng.read_negative_misses()
            logs = {"loss": self._loss_sum / max(self._loss_cnt, 1)}
            validate = (epoch >= (validation_burn_in - 1) and validation_data is not None
                        and (epoch + 1) % validation_freq == 0)
            if validate:
                self.is_fitted = True
                if val_findex is None:
                    val_findex = self._build_filter(validation_filter, lambda: self._index(validation_data))
                ranks = self.evaluate(validation_data, batch_size=validation_batch_size or batch_size, verbose=False,
                                      use_filter=validation_filter, corrupt_side=validation_corrupt_side,
                                      entities_subset=validation_entities_subset, dataset_type="valid",
                                      _filter_index=val_findex)
                logs.update({"val_mrr": mrr_score(ranks), "val_mr": mr_score(ranks),
                             "val_hits@1": hits_at_n_score(ranks, 1), "val_hits@10": hits_at_n_score(ranks, 10),
                             "val_hits@100": hits_at_n_score(ranks, 100)})
            history._log(epoch, logs)
            for cb in (callbacks or []):  # minimal Keras callback protocol: on_epoch_end + model.stop_training
                if hasattr(cb, "on_epoch_end"):
                    cb.on_epoch_end(epoch, logs)
            if verbose:
                print("Epoch %d/%d - " % (epoch + 1, epochs) + " - ".join("%s: %.4f" % kv for kv in logs.items()))
            if self.stop_training:
                break
        self.is_fitted = True
        self.history = history
        return history

    @staticmethod
    def _check_dropout(entity_dropout, relation_dropout, one_vs_all, k_vs_all):
        """The refusals of fit(entity_dropout=..., relation_dropout=...), before anything is indexed or trained: each a
        real, finite number in [0, 1) (not a bool), and a non-zero one needs one_vs_all or k_vs_all."""
        for name, p in (("entity_dropout", entity_dropout), ("relation_dropout", relation_dropout)):
            if (isinstance(p, bool) or not isinstance(p, numbers.Real) or not math.isfinite(p)
                    or not 0.0 <= p < 1.0):
                raise ValueError("%s must be a number in [0, 1), got %r" % (name, p))
        if (entity_dropout or relation_dropout) and one_vs_all is None and k_vs_all is None:
            raise ValueError("entity_dropout and relation_dropout apply to one_vs_all and k_vs_all training only: the "
                             "sampled training kernels (also with focusE or a user loss) do not apply them")

    def _uses_n3(self):
        return any(isinstance(r, regularizers.N3Regularizer) for r in self._regularizer)

    def _uses_dura(self):
        return any(isinstance(r, regularizers.DURARegularizer) for r in self._regularizer)

    def _check_per_occurrence(self, k_vs_all=None):
        """The refusals of a training call with a per-occurrence regulariser (N3, DURA), before anything is indexed or
        trained."""
        for name, used in (("N3", self._uses_n3()), ("DURA", self._uses_dura())):
            if not used:
                continue
            if k_vs_all is not None:
                raise NotImplementedError("the %s regularizer is not supported with k_vs_all: a KvsAll step has "
                                          "queries, not triples" % name)
            if self._world() > 1:
                raise NotImplementedError("the %s regularizer is single-GPU only" % name)

    def _per_occurrence_backward(self, batch):
        """The per-occurrence regulariser terms of this step's positives: N3 (KGEEngine.n3_backward) where a table has
        it with lambda > 0, and DURA (KGEEngine.dura_backward)."""
        if any(v > 0.0 for v in self.engine.n3_lambdas.values()):
            self.engine.n3_backward(batch, step=self._step)
        if self.engine.dura_weights is not None:
            self.engine.dura_backward(batch, step=self._step)

    def _check_reciprocal(self, call, one_vs_all=None, k_vs_all=None, focusE=False, relation_prediction_weight=0.0):
        """The refusals of a training call on a model with reciprocal relations, before anything is indexed or trained:
        only fit(one_vs_all=...) and fit(k_vs_all=...) train the inverse rows."""
        why = None
        if one_vs_all is None and k_vs_all is None:
            why = ("%s trains against sampled corruptions, whose fused kernels score both corruption sides of a positive "
                   "with its one relation row: use fit(one_vs_all=...) or fit(k_vs_all=...)" % call)
        elif focusE:
            why = "focusE is a sampled-training option"
        elif isinstance(self.compiled_loss, loss_functions.LossFunctionWrapper):
            why = "a user loss is a sampled-training option"
        elif (isinstance(relation_prediction_weight, numbers.Real) and not isinstance(relation_prediction_weight, bool)
              and relation_prediction_weight > 0):
            why = "the relation-prediction term is not defined for the inverse relations"
        elif self.distributed:
            why = "training is single-GPU only"
        if why is not None:
            raise NotImplementedError("reciprocal relations: %s" % why)

    def _check_negative_sampler(self, negative_sampler, filter_negatives, one_vs_all, k_vs_all, params=None):
        """The refusals of fit(negative_sampler=..., filter_negatives=..., negative_sampler_params=...), before anything
        is indexed or trained -> whether the step draws its corruptions with kge_sample_negatives or
        kge_nscaching_step ('uniform' without the filter does neither)."""
        if not isinstance(negative_sampler, str) or negative_sampler not in FIT_NEGATIVE_SAMPLERS:
            raise ValueError("negative_sampler must be one of %s, got %r"
                             % (", ".join(map(repr, FIT_NEGATIVE_SAMPLERS)), negative_sampler))
        if not isinstance(filter_negatives, bool):
            raise ValueError("filter_negatives must be a bool, got %r" % (filter_negatives,))
        if params is not None:
            self._check_nscaching_params(negative_sampler, params)
        if negative_sampler == "uniform" and not filter_negatives:
            return False
        if one_vs_all is not None or k_vs_all is not None:
            raise ValueError("negative_sampler and filter_negatives are sampled-training options: they cannot be "
                             "combined with one_vs_all or k_vs_all")
        if self._world() > 1:
            raise NotImplementedError("negative_sampler and filter_negatives are single-GPU only")
        return True

    def _check_shared_negatives(self, chunk, one_vs_all, k_vs_all, negative_sampler, filter_negatives, focusE):
        """The refusals of fit(shared_negatives=C), before anything is indexed or trained: C an int >= 0 (not a bool);
        C >= 1 needs sampled training on one GPU with a built-in loss, without focusE, and a sampler that picks only
        the side ('uniform' or 'bernoulli', unfiltered)."""
        if isinstance(chunk, (bool, np.bool_)) or not isinstance(chunk, (int, np.integer)) or chunk < 0:
            raise ValueError("shared_negatives must be an int >= 0 (positives per chunk; 0: off), got %r" % (chunk,))
        if chunk == 0:
            return
        if one_vs_all is not None or k_vs_all is not None:
            raise ValueError("shared_negatives is a sampled-training option: it cannot be combined with one_vs_all or "
                             "k_vs_all")
        if negative_sampler in ("pseudo_typed", "nscaching") or filter_negatives:
            raise ValueError("shared_negatives draws one candidate set per chunk, and negative_sampler=%r%s picks "
                             "entities per positive: use 'uniform' or 'bernoulli' without filter_negatives"
                             % (negative_sampler, " with filter_negatives=True" if filter_negatives else ""))
        if isinstance(self.compiled_loss, loss_functions.LossFunctionWrapper) or focusE:
            raise NotImplementedError("shared_negatives applies the compiled built-in loss inside its kernels: user "
                                      "losses and focusE are not supported")
        if self.distributed or self._world() > 1:
            raise NotImplementedError("shared_negatives is single-GPU only")

    @staticmethod
    def _check_nscaching_params(negative_sampler, params):
        """The refusals of negative_sampler_params: given with another sampler than 'nscaching', not a dict, unknown
        keys, values that are not ints (bools are refused) or out of bounds (N1, N2 >= 1, N1 + N2 <= 512)."""
        if negative_sampler != "nscaching":
            raise ValueError("negative_sampler_params applies to negative_sampler='nscaching' only, got sampler %r"
                             % (negative_sampler,))
        if not isinstance(params, dict):
            raise ValueError("negative_sampler_params must be a dict, got %r" % (params,))
        unknown = sorted(set(params) - set(NSCACHING_PARAMS), key=repr)
        if unknown:
            raise ValueError("unknown negative_sampler_params keys %s (known: %s)"
                             % (", ".join(map(repr, unknown)), ", ".join(map(repr, NSCACHING_PARAMS))))
        for key, v in params.items():
            if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)):
                raise ValueError("negative_sampler_params[%r] must be an int, got %r" % (key, v))
        p = dict(NSCACHING_PARAMS, **params)
        if p["cache_size"] < 1 or p["random_size"] < 1 or p["cache_size"] + p["random_size"] > NSCACHING_MAX_CANDIDATES:
            raise ValueError("negative_sampler_params needs cache_size >= 1, random_size >= 1 and cache_size + "
                             "random_size <= %d, got %d and %d"
                             % (NSCACHING_MAX_CANDIDATES, p["cache_size"], p["random_size"]))

    def _sampled_negatives(self, batch, sampler, start):
        """The corruptions of the sampled step on `batch` (fit's triples from `start`): None for the uniform draw of the
        training kernel, else the (repl, keep) views of kge_sample_negatives (a NegativeSamplerTables) or
        kge_nscaching_step (an NSCache)."""
        if sampler is None:
            return None
        if isinstance(sampler, NSCache):
            key_rows, update = sampler.batch(start, batch.shape[0])
            return self.engine.nscaching_negatives(batch, key_rows, update, sampler, self.seed, self._step)
        return self.engine.sample_negatives(batch, sampler, self.seed, self._step)

    def _sampled_step(self, batch, sampler=None, start=0):
        """One sampled training step on the device batch `batch`: on several GPUs this rank's share of the global-batch
        step (DataParallelTrainer), else the user loss's two-phase step, else the fused step, the per-occurrence
        regularisers and the optimizer.  sampler and start as in _sampled_negatives (None: the uniform draw)."""
        if self._world() > 1:
            self._dp.train_step(batch, None, seed=self.seed + 7919 * self._rank(), step=self._step)
        elif isinstance(self.compiled_loss, loss_functions.LossFunctionWrapper):
            self._user_loss_step(batch, sampler, start)
        else:
            negatives = self._sampled_negatives(batch, sampler, start)
            self.engine.forward_backward(batch, negatives, seed=self.seed, step=self._step, defer=True)
            self._per_occurrence_backward(batch)
            self.engine.apply_gradients()

    def _check_all_candidates(self, training, loss, focusE):
        """The refusals fit's all-candidate training types share: `training` ('1vsAll' or 'KvsAll') needs a trilinear
        model, the compiled loss `loss`, no focusE and one GPU."""
        if self.scoring_type not in ("DistMult", "ComplEx", "HolE"):
            raise NotImplementedError("%s training is implemented for DistMult, ComplEx and HolE (inner-product "
                                      "scores), not for %s" % (training, self.scoring_type))
        if isinstance(self.compiled_loss, loss_functions.LossFunctionWrapper) or self.compiled_loss.name != loss:
            raise ValueError("%s training needs the loss %r, got %r" % (training, loss, self.compiled_loss.name))
        if focusE:
            raise NotImplementedError("%s training does not support focusE" % training)
        if self._world() > 1:
            raise NotImplementedError("%s training is single-GPU only" % training)

    def _check_one_vs_all(self, one_vs_all, focusE):
        """The refusals of fit(one_vs_all=...), before anything is indexed or trained."""
        if not isinstance(one_vs_all, str) or one_vs_all not in _lib.ONE_VS_ALL_SIDES:
            raise ValueError("one_vs_all must be None, 's,o', 'o' or 's', got %r" % (one_vs_all,))
        self._check_all_candidates("1vsAll", "multiclass_nll", focusE)

    def _check_k_vs_all(self, k_vs_all, label_smoothing, one_vs_all, focusE):
        """The refusals of fit(k_vs_all=..., label_smoothing=...), before anything is indexed or trained."""
        if k_vs_all is not None:
            if not isinstance(k_vs_all, str) or k_vs_all not in _lib.ONE_VS_ALL_SIDES:
                raise ValueError("k_vs_all must be None, 's,o', 'o' or 's', got %r" % (k_vs_all,))
            if one_vs_all is not None:
                raise ValueError("k_vs_all and one_vs_all are two training types: give one of them")
        if (isinstance(label_smoothing, bool) or not isinstance(label_smoothing, numbers.Real)
                or not math.isfinite(label_smoothing) or not 0.0 <= label_smoothing < 1.0):
            raise ValueError("label_smoothing must be a number in [0, 1), got %r" % (label_smoothing,))
        if k_vs_all is None:
            raise ValueError("label_smoothing applies to KvsAll training only (k_vs_all=...)")
        self._check_all_candidates("KvsAll", "nll", focusE)

    @staticmethod
    def _check_relation_prediction(weight, one_vs_all, k_vs_all):
        """The refusals of fit(relation_prediction_weight=...), before anything is indexed or trained (n_rel >= 2 is
        checked once the relations are indexed)."""
        if (isinstance(weight, bool) or not isinstance(weight, numbers.Real) or not math.isfinite(weight)
                or weight < 0):
            raise ValueError("relation_prediction_weight must be a finite number >= 0, got %r" % (weight,))
        if weight > 0 and k_vs_all is not None:
            raise ValueError("relation_prediction_weight is a 1vsAll term: it cannot be combined with k_vs_all")
        if weight > 0 and one_vs_all is None:
            raise ValueError("relation_prediction_weight needs 1vsAll training (one_vs_all=...)")

    def _k_vs_all_step(self, kva, ranges, label_smoothing):
        """One KvsAll step: the query rows [lo, hi) of side o and of side s (ranges, from k_vs_all_steps), then the
        optimizer."""
        for side, (lo, hi) in zip(("o", "s"), ranges):
            if hi > lo:
                q, off, ids = kva[side]
                self.engine.k_vs_all_backward(q[lo:hi], "o" if self.reciprocal_relations else side, off[lo:hi + 1],
                                              ids, label_smoothing, step=self._step)
        self.engine.apply_gradients()

    def train_on_batch(self, x):
        """Keras Model.train_on_batch (the reference model is a tf.keras.Model): one train_step on ONE
        host batch -- H2D copy of the batch, fused step, D2H read of the batch loss, which is returned.
        x: [B,3] raw triples (numpy) or an int32 torch tensor of already indexed ids (pinned for speed)."""
        self._assert_compile_was_called()
        if self.reciprocal_relations:
            self._check_reciprocal("train_on_batch")
        self._check_per_occurrence()
        if torch.is_tensor(x):
            host = x
        else:
            host = torch.as_tensor(self._index(x, fit=self.engine is None))
        if self.engine is None:
            if self.data_indexer is not False:
                self.max_ent_size = self.data_indexer.get_entities_count()
                self.max_rel_size = self.data_indexer.get_relations_count()
            self._build_engine()
        # on several GPUs x is this rank's share of the global batch; gradients are exchanged inside the step
        self._sampled_step(host.to(self.engine.device, non_blocking=True))
        self._step += 1
        if self._world() > 1:
            self._dp.reduce_loss_()  # the loss of the GLOBAL batch, identical on every rank
        loss = self.engine.read_loss()
        self._loss_sum += loss
        self._loss_cnt += 1
        self.is_fitted = True
        return loss

    def train_on_batches(self, batches, prefetch=2):
        """Streamed training from HOST memory: one train_step per batch of `batches` (an iterable of [B,3] int32 id
        arrays, numpy or torch; the tf.data generator path of the reference's fit, graph_data_loader.py:472-523,:760-766
        with its prefetch(2)).  Every step copies ITS batch host->device and reads ITS loss device->host, but nothing
        blocks: batch i+1 travels on a copy stream through a persistent pinned ring while step i runs, and the 16-byte
        loss record of step i is copied asynchronously and read one step later.  Returns the list of per-batch losses."""
        self._assert_compile_was_called()
        if self.reciprocal_relations:
            self._check_reciprocal("train_on_batches")
        self._check_per_occurrence()
        it = iter(batches)
        first = next(it, None)
        if first is None:
            return []
        as_host = lambda x: x if torch.is_tensor(x) else torch.as_tensor(np.ascontiguousarray(x, dtype=np.int32))
        first = as_host(first)
        if self.engine is None:
            if self.max_ent_size is None or self.max_rel_size is None:
                raise ValueError("train_on_batches needs max_ent_size/max_rel_size (ids are already indexed)")
            self._build_engine()
        eng = self.engine
        if getattr(self, "hot_entities_from", None) is not None:  # streamed training sees no training set to count: an indexed
            eng.set_hot_entities(triples=self.hot_entities_from)   # [N,3] array may be attached for the hot-entity hint of fit()
            self.hot_entities_from = None
        dev = eng.device
        depth = max(2, int(prefetch))
        cap = first.shape[0]
        main = torch.cuda.current_stream(dev)
        if getattr(self, "_pipe", None) is None or self._pipe["cap"] < cap or self._pipe["depth"] != depth:
            self._pipe = {"cap": cap, "depth": depth, "copy": torch.cuda.Stream(dev),
                          "pin": [torch.empty((cap, 3), dtype=torch.int32).pin_memory() for _ in range(depth)],
                          "dev": [torch.empty((cap, 3), dtype=torch.int32, device=dev) for _ in range(depth)],
                          "ready": [torch.cuda.Event() for _ in range(depth)], "free": [torch.cuda.Event() for _ in range(depth)],
                          "loss_pin": torch.zeros((depth, 2), dtype=torch.float64).pin_memory(),
                          "loss_ev": [torch.cuda.Event() for _ in range(depth)]}
            for e in self._pipe["free"]:
                e.record(main)
        P = self._pipe
        copy = P["copy"]

        def stage(i, hb):  # host batch -> (pinned ring slot ->) device ring slot, on the copy stream; never blocks on a STEP
            s = i % depth
            n = hb.shape[0]
            if n > P["cap"]:
                raise ValueError("batch of %d positives exceeds the first batch (%d) this pipeline was sized for" % (n, P["cap"]))
            if hb.is_pinned():
                src = hb
            else:
                P["ready"][s].synchronize()  # the previous H2D copy OUT of this pinned slot has finished (not the step)
                P["pin"][s][:n].copy_(hb)
                src = P["pin"][s][:n]
            copy.wait_event(P["free"][s])    # stream-ordered: the step that read this device slot last is done
            with torch.cuda.stream(copy):
                P["dev"][s][:n].copy_(src, non_blocking=True)
                P["ready"][s].record(copy)
            return s, n

        losses, pending = [], []  # pending: (slot, cumulative-loss record not yet read)
        eng.loss_acc.zero_()  # the accumulator is cumulative from here on; per-step losses are differences of records
        prev_total = 0.0
        queued = [stage(0, first)]
        i = 0
        while queued:
            nxt = next(it, None)
            if nxt is not None:
                queued.append(stage(i + 1, as_host(nxt)))  # overlaps step i
            s, n = queued.pop(0)
            main.wait_event(P["ready"][s])
            self._sampled_step(P["dev"][s][:n])
            P["free"][s].record(main)
            P["loss_pin"][s].copy_(eng.loss_acc, non_blocking=True)  # D2H of this step's (cumulative) loss record
            P["loss_ev"][s].record(main)
            pending.append(s)
            if len(pending) >= depth:  # read the record of step i-depth+1 (long complete) before its slot is reused
                ps = pending.pop(0)
                P["loss_ev"][ps].synchronize()
                tot = float(P["loss_pin"][ps].sum())
                losses.append(tot - prev_total)
                prev_total = tot
            self._step += 1
            self._loss_cnt += 1
            i += 1
        for ps in pending:
            P["loss_ev"][ps].synchronize()
            tot = float(P["loss_pin"][ps].sum())
            losses.append(tot - prev_total)
            prev_total = tot
        eng.loss_acc.zero_()
        self._loss_sum += sum(losses)
        self.is_fitted = True
        return losses

    def _user_loss_step(self, batch, sampler=None, start=0):
        self._two_phase_step(batch, None, sampler, start)

    def _two_phase_step(self, batch, weights, sampler=None, start=0):
        """LossFunctionWrapper / FocusE path: scores from the kernel, dL/dscore from torch autograd
        over a handful of elementwise ops, gradients from the kernel again.  sampler: the fit's NegativeSamplerTables or
        NSCache (batch = the fit's triples from `start`), or None for the uniform corruptions."""
        eng, B = self.engine, batch.shape[0]
        if sampler is not None:
            repl, keep = self._sampled_negatives(batch, sampler, start)
        else:
            neg = eng.generate_corruptions(batch, self.seed, self._step)
            tiled = batch.repeat(self.eta, 1)
            keep = (neg[:, 0] == tiled[:, 0]).to(torch.uint8).contiguous()
            repl = torch.where(keep.bool(), neg[:, 2], neg[:, 0]).contiguous()
        sp = torch.empty(B, dtype=torch.float32, device=eng.device)
        sn = torch.empty(B * self.eta, dtype=torch.float32, device=eng.device)
        eng.forward_backward(batch, (repl, keep), seed=self.seed, step=self._step, mode=_lib.STEP_FORWARD_ONLY,
                             scores_pos=sp, scores_neg=sn)
        spg, sng = sp.requires_grad_(True), sn.requires_grad_(True)
        fp, fn = spg, sng
        if weights is not None:  # compute_focusE_weights (:342-368) + score re-weighting (:396-406)
            w = weights.mean(1)
            sw = self._focuse_sw
            fp = self._focuse_nl(spg) * (sw + (1 - sw) * (1 - w))
            fn = self._focuse_nl(sng) * (sw + (1 - sw) * w.repeat(self.eta))
        if isinstance(self.compiled_loss, loss_functions.LossFunctionWrapper):
            loss = self.compiled_loss._user_losses(fp, fn.reshape(self.eta, -1)).sum()
        else:
            from .torch_losses import per_positive_loss
            name, lp = self.compiled_loss.kernel_params()
            loss = per_positive_loss(name, fp, fn.reshape(self.eta, -1), lp).sum()
        loss.backward()
        eng.forward_backward(batch, (repl, keep), seed=self.seed, step=self._step, mode=_lib.STEP_BACKWARD_EXT,
                             dpos=spg.grad.contiguous(), dneg=sng.grad.contiguous())  # step: the lazy rule's row stamp
        self._per_occurrence_backward(batch)
        eng.apply_gradients()
        eng.loss_acc[0] += loss.detach().double()

    # ------------------------------------------------------------------ predict
    def predict(self, x, batch_size=32, verbose=0, callbacks=None):
        """predict (:1736-1823): fp32 scores; triples with unknown labels are dropped."""
        if not self.is_fitted:
            raise RuntimeError("Model has not been fitted.")
        t = self._index(x)
        if len(t) == 0:
            return np.zeros(0, np.float32)
        return self.engine.score(self._to_dev(t, np.int32)).cpu().numpy()

    # ------------------------------------------------------------------ evaluate
    def _build_filter(self, use_filter, indexed_x):
        """FilterIndex of evaluate's use_filter: a dict of datasets (train/valid/test), or True for the evaluated data
        itself (indexed_x() returns it indexed); None for no filter."""
        if not (isinstance(use_filter, dict) or use_filter is True):
            return None
        parts = [indexed_x()] if use_filter is True else [self._index(v) for v in use_filter.values()]
        return FilterIndex(np.concatenate(parts), self.max_ent_size)

    def evaluate(self, x=None, batch_size=10, verbose=True, use_filter=False, corrupt_side="s,o",
                 entities_subset=None, ranking_strategy="worst", callbacks=None, dataset_type="test", _filter_index=None):
        """evaluate (:1516-1692) -> int32 ranks [n, 2] for 's,o', [n, 1] otherwise.
        corrupt_side='p' (extension: relation prediction) ranks each triple's relation among all relations for its
        (s, o), by the same count, ranking_strategy and use_filter rules (a known (s, r, o) removes r); entities_subset
        does not apply to it.  `batch_size` only lower-bounds the device chunk: results do not depend on it.
        With reciprocal relations, side s of (s, p, o) is ranked as side o of (o, p^-1, s) with the same filter and
        candidates, and corrupt_side='p' ranks among the forward relations only.
        _filter_index: the FilterIndex that use_filter would build (_build_filter), when the caller keeps one across calls
        (fit's validations)."""
        assert corrupt_side in ["s", "o", "s,o", "s+o", "p"], "Invalid value for corrupt_side"
        assert ranking_strategy in ["best", "middle", "worst"], "Invalid value for ranking_strategy"
        if corrupt_side == "p" and entities_subset is not None:
            raise ValueError("entities_subset does not apply to corrupt_side='p': the candidates are the relations")
        if not self.is_fitted:
            raise RuntimeError("Model has not been fitted.")
        if self.reciprocal_relations and self._world() > 1:
            raise NotImplementedError("reciprocal relations: evaluate is single-GPU only")
        eng = self.engine
        t = self._index(x)
        n = len(t)
        sides = ["p"] if corrupt_side == "p" else [s for s in ("s", "o") if s in corrupt_side]
        # candidates: all entities or a subset (:1634-1643)
        cand_ids, position_of = None, None
        if entities_subset is not None:
            sub = self.get_indexes(np.asarray(entities_subset), "e") if self.data_indexer is not False \
                else np.asarray(entities_subset, np.int32)
            cand_ids = self._to_dev(sub, np.int32)
            position_of = np.full(self.max_ent_size, -1, np.int64)
            position_of[sub] = np.arange(len(sub))
        findex = _filter_index if _filter_index is not None else self._build_filter(use_filter, lambda: t)
        out = np.zeros((n, len(sides)), np.int32)
        chunk = max(int(batch_size), 4096)
        for start in range(0, n, chunk):
            tb = t[start:start + chunk]
            td = self._to_dev(tb, np.int32)
            for j, side in enumerate(sides):
                off = idx = None
                if findex is not None:
                    o_np, i_np = findex.lookup(tb, side, position_of)
                    off, idx = self._to_dev(o_np, np.int64), self._to_dev(i_np, np.int32)
                if self.reciprocal_relations and side != "o":
                    # side s: the side-o rank of the inverse (o, p^-1, s), with the same filter list; side p: among the
                    # forward relations only
                    rd, rs, n_rel = (td, "p", self.max_rel_size) if side == "p" else \
                        (self._to_dev(reciprocal_triples(tb, self.max_rel_size, "s"), np.int32), "o", None)
                    r = eng.rank(rd, rs, ranking_strategy, off, idx, cand_ids=cand_ids, n_cand=n_rel)
                elif self._world() > 1 and cand_ids is None and side != "p":
                    # row-sharded candidates: RAW counters summed over ranks, tie strategy applied once ('middle' is not
                    # additive over partitions, AbstractScoringLayer.py:232-244); the relation side runs on each rank
                    # locally (the relation table is replicated)
                    from ..parallel import allreduce_sum_, row_shard
                    lo, hi = row_shard(self.max_ent_size, self._world(), self._rank())
                    cnt = torch.zeros((len(tb), 3), dtype=torch.int32, device=eng.device)
                    eng.rank(td, side, ranking_strategy, off, idx, cand_begin=lo, n_cand=hi - lo, counts=cnt)
                    allreduce_sum_([cnt])
                    r = eng.finalize_ranks(cnt, ranking_strategy)
                else:
                    r = eng.rank(td, side, ranking_strategy, off, idx, cand_ids=cand_ids)
                out[start:start + len(tb), j] = r.cpu().numpy()
        if corrupt_side == "s+o":  # :1459-1463 sum BEFORE the +1
            out = out.sum(1, keepdims=True)
        return (out + 1).astype(np.int32)  # :1684

    # ------------------------------------------------------------------ calibration
    def calibrate(self, X_pos, X_neg=None, positive_base_rate=None, batch_size=32, epochs=50, verbose=0):
        """calibrate (:1922-2122) with CalibrationLayer (layers/calibration/calibrate.py:11-129): Platt scaling,
        two scalars (w, b) fitted with Adam on the kernel's scores of positives and negatives (given, or
        generated corruptions when only positive_base_rate is given)."""
        if not self.is_fitted:
            raise RuntimeError("Model has not been fitted.")
        self.is_calibrated = False
        pos = self._to_dev(self._index(X_pos), np.int32)
        pos_size = pos.shape[0]
        with_corruption = X_neg is None
        if with_corruption:
            assert positive_base_rate is not None, "Please provide the negatives or positive base rate!"
            neg, neg_size = None, pos_size
        else:
            neg = self._to_dev(self._index(X_neg), np.int32)
            neg_size = neg.shape[0]
            if positive_base_rate is None:
                positive_base_rate = pos_size / (pos_size + neg_size)
        if positive_base_rate is not None and (positive_base_rate <= 0 or positive_base_rate >= 1):
            raise ValueError("positive_base_rate must be a value between 0 and 1.")
        dev = self.engine.device
        w = torch.zeros((), device=dev, requires_grad=True)  # calibrate.py:60-63
        b = torch.tensor(float(np.log((neg_size + 1.0) / (pos_size + 1.0))), device=dev, requires_grad=True)
        opt = torch.optim.Adam([w, b], lr=1e-3, eps=1e-7)
        n_batches = int(np.ceil(pos_size / batch_size))
        nb_size = int(np.ceil(neg_size / n_batches)) if not with_corruption else None
        step = 0
        for _ in range(epochs):
            for i in range(n_batches):
                pb = pos[i * batch_size:(i + 1) * batch_size].contiguous()
                sp = self.engine.score(pb)
                if with_corruption:  # ONE corruption per positive (eta=1, :1886): the j=0 block of the tile-ordered tensor
                    sn = self.engine.score(self.engine.generate_corruptions(pb, self.seed, step)[:pb.shape[0]].contiguous())
                else:
                    sn = self.engine.score(neg[i * nb_size:(i + 1) * nb_size].contiguous())
                step += 1
                scores = torch.cat([sp, sn])
                logits = -(w * scores + b)
                labels = torch.cat([torch.full_like(sp, (pos_size + 1.0) / (pos_size + 2.0)),
                                    torch.full_like(sn, 1.0 / (neg_size + 2.0))])
                weights = torch.cat([torch.full_like(sp, sn.shape[0] / max(sp.shape[0], 1)),
                                     torch.full_like(sn, (1.0 - positive_base_rate) / positive_base_rate)])
                loss = (weights * torch.nn.functional.binary_cross_entropy_with_logits(logits, labels, reduction="none")).mean()
                opt.zero_grad()
                loss.backward()
                opt.step()
        self.calib_w, self.calib_b = float(w.detach()), float(b.detach())
        self.is_calibrated = True

    def predict_proba(self, x, batch_size=32, verbose=0, callbacks=None):
        """predict_proba (:2124-2212): sigmoid(-(w*score + b)) of the calibrated model."""
        if not self.is_calibrated:
            raise RuntimeError("Model has not been calibrated. Please call `model.calibrate(...)` before predicting probabilities.")
        sc = self.predict(x, batch_size=batch_size)
        return (1.0 / (1.0 + np.exp(self.calib_w * sc + self.calib_b))).astype(np.float32)

    # ------------------------------------------------------------------ embeddings / weights
    def get_embeddings(self, entities, embedding_type="e"):
        """get_embeddings (:2214): rows of the dense [rows, internal_k] tables.  embedding_type 'e' (entities), 'r'
        (relations; with reciprocal relations the forward rows) or 'r_inv' (extension: the inverse rows of the given
        relations, on a model with reciprocal relations only)."""
        if not self.is_fitted:
            raise RuntimeError("Model has not been fitted.")
        if embedding_type not in ("e", "r", "r_inv"):
            raise ValueError("Invalid entity type: %s" % embedding_type)
        if embedding_type == "r_inv" and not self.reciprocal_relations:
            raise ValueError("embedding_type 'r_inv' needs a model with reciprocal relations")
        ent, rel = self.engine.get_embeddings()
        kind = "e" if embedding_type == "e" else "r"
        idx = self.get_indexes(np.asarray(entities), kind) if self.data_indexer is not False \
            else np.asarray(entities, np.int64)
        if embedding_type == "r_inv":
            idx = np.asarray(idx, np.int64) + self.max_rel_size
        table = ent if embedding_type == "e" else rel
        return table[torch.as_tensor(idx, dtype=torch.long, device=table.device)].cpu().numpy()

    def _snapshot_tables(self):
        """Device copies of the live entity and relation tables (what Keras's get_weights returns for the reference:
        no optimizer slots, no step count).  engine.ent / engine.rel view whichever parameter block is current, also
        after the deferred steps swapped the engine's two blocks."""
        return self.engine.ent.clone(), self.engine.rel.clone()

    def _restore_tables(self, snapshot):
        """Write a _snapshot_tables() copy back into the live tables."""
        self.engine.ent.copy_(snapshot[0])
        self.engine.rel.copy_(snapshot[1])

    def save_weights(self, filepath):
        """Tables + optimizer slots and state (step count, Nadam's momentum cache) + indexer in one pickle (the
        reference's Keras format is TF-specific)."""
        ent, rel = self.engine.get_embeddings()
        state = {"ent": ent.cpu().numpy(), "rel": rel.cpu().numpy(), "t": self.engine.t, "step": self._step,
                 "nadam_cache": float(getattr(self.engine, "nadam_cache", 1.0)),
                 "slots": {k: [None if s is None else s.cpu().numpy() for s in v] for k, v in self.engine.slots.items()},
                 "indexer": self.data_indexer, "max_ent_size": self.max_ent_size, "max_rel_size": self.max_rel_size,
                 "reciprocal_relations": self.reciprocal_relations}
        with open(filepath, "wb") as f:
            pickle.dump(state, f)

    def load_weights(self, filepath):
        self._assert_compile_was_called()
        with open(filepath, "rb") as f:
            state = pickle.load(f)
        saved = state.get("reciprocal_relations", False)  # files written before the flag existed have none
        if saved != self.reciprocal_relations:
            raise ValueError("the weights were saved by a model with reciprocal_relations=%s, this model has %s"
                             % (saved, self.reciprocal_relations))
        self.data_indexer = state["indexer"]
        self.max_ent_size, self.max_rel_size = state["max_ent_size"], state["max_rel_size"]
        self._build_engine()
        self.engine.set_embeddings(state["ent"], state["rel"])
        self.engine.t, self._step = state["t"], state["step"]
        # Nadam's momentum cache (an fp32 value, exact as a float); files written before Nadam have none
        self.engine.nadam_cache = np.float32(state.get("nadam_cache", 1.0))
        for k, v in state["slots"].items():
            for n, s in enumerate(v):
                if s is not None:
                    self.engine.slots[k][n].copy_(torch.as_tensor(s))
        self.is_fitted = True
