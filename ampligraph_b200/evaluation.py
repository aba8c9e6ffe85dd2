"""Rank metrics (mirror of ampligraph/evaluation/metrics.py:18-259): O(n) numpy on the
int32 ranks the ranking kernel returns.

The evaluation protocol of ampligraph/evaluation/protocol.py is here too, on the host: train_test_split_no_unseen,
filter_unseen_entities and select_best_model_ranking.  Their arithmetic is the training step and the ranking kernel
behind ScoringBasedEmbeddingModel.fit / evaluate; what is here only splits data and sequences candidates.
Deviations from the reference are listed in DESIGN.md §7.
"""
import logging
import operator
from collections.abc import Iterable
from contextlib import contextmanager
from itertools import islice, product

import numpy as np
import pandas as pd

logger = logging.getLogger(__name__)


def _flat(ranks):
    r = np.asarray(ranks).reshape(-1)
    return r


def mrr_score(ranks):
    """Mean reciprocal rank (metrics.py:155)."""
    r = _flat(ranks)
    return float(np.sum(1.0 / r) / len(r))


def mr_score(ranks):
    """Mean rank (metrics.py:196)."""
    r = _flat(ranks)
    return float(np.sum(r) / len(r))


def hits_at_n_score(ranks, n):
    """Hits@n (metrics.py:18)."""
    r = _flat(ranks)
    return float(np.sum(r <= n) / len(r))


def rank_score(y_true, y_pred, pos_lab=1):
    """Rank of the positive among y_pred (metrics.py:87)."""
    y_true, y_pred = np.asarray(y_true), np.asarray(y_pred)
    idx = np.argsort(y_pred)[::-1]
    return int(np.where(y_true[idx] == pos_lab)[0][0] + 1)


# ---------------------------------------------------------------------------------------------------- splitting
SPLIT_ERROR = ("Cannot create a test split of the desired size. Some entities will not occur in both training and test "
               "set. Set allow_duplication=True,remove filter on test predicates or set test_size to a smaller value.")


def _split_accepted(el):
    """Which triples the reference's counting walk (protocol.py:136-165) puts in the test set if it never stops early.
    el: [n, 3] int64 element ids (s, p, o) of the triples in walk order, entities and relations in one id space.  See
    train_test_split_no_unseen for why this equals the walk."""
    n = len(el)
    pos = np.arange(n)
    last = np.full(int(el.max(initial=-1)) + 1, -1, np.int64)
    np.maximum.at(last, el.reshape(-1), np.repeat(pos, 3))
    at_last = last[el] == pos[:, None]  # [n, 3]: this position is the last occurrence of that element
    accepted = np.ones(n, bool)
    has_rejected = np.zeros(len(last), bool)
    cand = np.flatnonzero(at_last.any(1))
    for i, (x, l) in zip(cand.tolist(), zip(el[cand].tolist(), at_last[cand].tolist())):
        if (l[0] and not has_rejected[x[0]]) or (l[1] and not has_rejected[x[1]]) or (l[2] and not has_rejected[x[2]]):
            accepted[i] = False
            has_rejected[x] = True
    return accepted


def train_test_split_no_unseen(X, test_size=100, seed=0, allow_duplication=False, filtered_test_predicates=None):
    """Split X into (X_train, X_test) so that every entity and relation of X_test also occurs in X_train
    (protocol.py:27-198): the same arrays, row for row, as the reference for every input, or the same error.

    X: ndarray [n, 3].  test_size: number of test triples, or a float fraction of the candidates (int(n * test_size)).
    allow_duplication: when fewer triples can be taken, fill the test set with repeats drawn from it instead of raising.
    filtered_test_predicates: only triples with these predicates are test candidates; the others go to X_train first.

    The random stream is the reference's (`permutation` of the candidates, `choice` for the repeats, then one
    `permutation` of each result) drawn from a local np.random.RandomState(seed): the global numpy generator is neither
    reseeded nor advanced.

    The reference walks the shuffled candidates with a count per element (entity or relation), rem_x, set to the
    occurrences of x in the candidates (a self-loop's entity counts twice).  A triple takes its elements' occurrences off
    the counts; it goes to the test set if every count stays above zero, else it goes to train and its occurrences are
    put back.  The walk stops at the test_size-th test triple, and every triple after it goes to train.  This function
    computes the same walk without visiting every triple:

    * Before position i, rem_x is the number of occurrences of x in the rejected positions before i and in all the
      positions from i on (induction: an accepted triple removes its own occurrences, a rejected one puts them back).
      So triple i is rejected exactly when one of its elements x occurs neither in an earlier rejected position nor in a
      later position.
    * A position that is not the last occurrence of any of its elements is therefore always accepted, and a position i
      that is the last occurrence of x is rejected because of x exactly when no earlier occurrence of x was rejected.
    * Rejections happen only at last occurrences, of which there are at most n_ent + n_rel.  Walking those positions in
      order with one "x has a rejected occurrence" flag per element gives every decision; a rejection sets the flag of
      all three elements of its triple.
    * The early stop only truncates the walk, since a decision depends on earlier decisions only: the test set is the
      accepted positions up to the test_size-th acceptance (found with a cumsum), and the train set is the rejected
      positions before it followed by every position after it, which is the reference's order.  Without that many
      acceptances the walk runs to the end and the reference's shortfall rule (repeats or the error) applies.
    """
    rs = np.random.RandomState(seed)
    if filtered_test_predicates:
        is_cand = np.isin(X[:, 1], filtered_test_predicates)
        C, X_train = X[is_cand], X[~is_cand]
    else:
        C, X_train = X, None
    if isinstance(test_size, float):
        test_size = int(len(C) * test_size)
    order = rs.permutation(np.arange(C.shape[0]))
    # element ids by hashing (pd.factorize: the same equality as the reference's np.unique, without its sort)
    ent, _ = pd.factorize(np.concatenate([C[:, 0], C[:, 2]]), use_na_sentinel=False)
    rel, _ = pd.factorize(C[:, 1], use_na_sentinel=False)
    n_ent = int(ent.max(initial=-1)) + 1
    el = np.stack([ent[:len(C)], n_ent + rel, ent[len(C):]], 1).astype(np.int64)
    accepted = _split_accepted(el[order])
    pos = np.arange(len(order))
    n_acc = int(accepted.sum())
    if 1 <= test_size <= n_acc and test_size == int(test_size):  # the walk stops at the test_size-th acceptance
        cut = int(np.searchsorted(np.cumsum(accepted), test_size))
        idx_test = order[accepted & (pos <= cut)]
        idx_train = order[(~accepted & (pos < cut)) | (pos > cut)]
    else:
        idx_test, idx_train = order[accepted], order[~accepted]
        if n_acc != test_size:
            if not allow_duplication:
                raise Exception(SPLIT_ERROR)
            extra = rs.choice(idx_test.tolist(), size=(test_size - n_acc))
            idx_test = np.concatenate([idx_test, np.asarray(extra, dtype=idx_test.dtype)])
    X_train = C[idx_train] if X_train is None else np.concatenate([X_train, C[idx_train]])
    X_test = C[idx_test]
    return rs.permutation(X_train), rs.permutation(X_test)


def filter_unseen_entities(X, model, verbose=False):
    """Keep the triples of X whose subject and object the model has seen in training (protocol.py:201-233); X itself
    when nothing is removed.  The seen entities are those of the model's DataIndexer, or the ids below max_ent_size for
    a model trained with use_indexer=False (integer ids)."""
    if model.data_indexer is False:
        ids = np.asarray(X)
        seen = lambda col: (ids[:, col] >= 0) & (ids[:, col] < model.max_ent_size)
    elif not isinstance(model.data_indexer, bool):
        index = model.data_indexer._ent_index
        seen = lambda col: index.get_indexer(np.asarray(X)[:, col]) >= 0
    else:
        raise RuntimeError("Model has not been fitted.")
    df = pd.DataFrame(X, columns=["s", "p", "o"])
    keep = seen(0) & seen(2)
    n_removed = int(len(df) - keep.sum())
    if n_removed > 0:
        msg = "Removing {} triples containing unseen entities. ".format(n_removed)
        if verbose:
            logger.info(msg)
        logger.debug(msg)
        return df[keep].values
    return X


# ---------------------------------------------------------------------------------------------------- model selection
def _flatten(grid):
    """{"a": {"b": v}} -> {("a", "b"): v}: the keys whose values are not dicts first, in order, then the nested ones."""
    flat = {k: v for k, v in grid.items() if not isinstance(v, dict)}
    for nk, sub in grid.items():
        if isinstance(sub, dict):
            flat.update({(nk, k): v for k, v in sub.items()})
    return flat


def _unflatten(flat):
    """Inverse of _flatten: tuple keys (outer, inner) become nested dicts, which replace a plain key of the same name."""
    nested = {}
    for k, v in flat.items():
        if isinstance(k, tuple):
            nested.setdefault(k[0], {})[k[1]] = v
    return {**{k: v for k, v in flat.items() if not isinstance(k, tuple)}, **nested}


def _param_key(param):
    """What the reference hashes to recognise a combination it has already tried (_get_param_hash)."""
    return frozenset(_flatten(_unflatten(param)).items())


def _grid_combinations(grid):
    """Every combination of a grid of lists, first key slowest, without repeats (_next_hyperparam)."""
    flat = _flatten(grid)
    seen = set()
    for values in product(*flat.values()):
        param = dict(zip(flat.keys(), values))
        key = _param_key(param)
        if key not in seen:
            seen.add(key)
            yield _unflatten(param)


def _sample(grid):
    """One random combination (_sample_parameters): callables are called, lists drawn from with np.random.choice
    (an int64 draw becomes int32), nested dicts sampled in turn, anything else kept."""
    param = {}
    for k, v in grid.items():
        if callable(v):
            param[k] = v()
        elif isinstance(v, dict):
            param[k] = _sample(v)
        elif isinstance(v, Iterable) and not isinstance(v, str):
            draw = np.random.choice(v)
            param[k] = draw.astype(np.int32) if isinstance(draw, np.int64) else draw
        else:
            param[k] = v
    return param


@contextmanager
def _global_stream(rs):
    """Run with rs's state as numpy's global generator, so that np.random.choice and the user's callables of a grid
    (e.g. lambda: np.random.uniform(...)) draw the reference's stream, then hand the state back to rs and restore the
    caller's global state."""
    saved = np.random.get_state()
    np.random.set_state(rs.get_state())
    try:
        yield
    finally:
        rs.set_state(np.random.get_state())
        np.random.set_state(saved)


def _random_combinations(grid, rs):
    """Random combinations without repeats (_next_hyperparam_random), drawn from rs."""
    seen = set()
    while True:
        with _global_stream(rs):
            param = _sample(grid)
        key = _param_key(param)
        if key not in seen:
            seen.add(key)
            yield param


def _lists_from_scalars(grid):
    """A copy of grid with every scalar (or string) value, nested ones included, wrapped in a one-element list
    (_scalars_into_lists); lists, callables and other iterables are kept as they are."""
    out = {}
    for k, v in grid.items():
        if isinstance(v, dict):
            out[k] = _lists_from_scalars(v)
        elif isinstance(v, str) or not (callable(v) or isinstance(v, Iterable)):
            out[k] = [v]
        else:
            out[k] = v
    return out


def _combinations(model_class, param_grid, max_combinations, param_grid_random_seed):
    """(combinations, how many) for select_best_model_ranking, on a copy of param_grid with model_name added last."""
    grid = _lists_from_scalars({**param_grid, "model_name": model_class})
    total = 1
    for v in grid.values():
        if isinstance(v, list):
            total *= len(v)
        elif isinstance(v, dict):
            total *= int(np.prod([len(x) for x in v.values() if isinstance(x, list)]))
    if max_combinations is None:
        return _grid_combinations(grid), total
    n = np.min([total, max_combinations])
    return islice(_random_combinations(grid, np.random.RandomState(param_grid_random_seed)), n), n


def _as_int32(v):
    """The reference takes eta as `.astype(np.int32)`, which only numpy scalars have; a Python int is accepted too."""
    return v.astype(np.int32) if isinstance(v, np.generic) else operator.index(v)


def _build_model(model_class, params, eta):
    from .latent_features import ScoringBasedEmbeddingModel
    from .latent_features import loss_functions, optimizers, regularizers
    model = ScoringBasedEmbeddingModel(eta=eta, k=params.get("k", 100), scoring_type=model_class,
                                       reciprocal_relations=params.get("reciprocal_relations", False))
    model.compile(optimizer=optimizers.get(params.get("optimizer", "adam"), params.get("optimizer_params", {})),
                  loss=loss_functions.get(params.get("loss", "multiclass_nll"), params.get("loss_params", {})),
                  entity_relation_regularizer=regularizers.get(params.get("regularizer"),
                                                               params.get("regularizer_params", {})),
                  entity_relation_initializer=params.get("initializer", "glorot_uniform"))
    return model


def _metrics(ranks):
    return {"mrr": mrr_score(ranks), "mr": mr_score(ranks), "hits_1": hits_at_n_score(ranks, n=1),
            "hits_3": hits_at_n_score(ranks, n=3), "hits_10": hits_at_n_score(ranks, n=10)}


def select_best_model_ranking(model_class, X_train, X_valid, X_test, param_grid, max_combinations=None,
                              param_grid_random_seed=0, use_filter=True, early_stopping=True, early_stopping_params=None,
                              use_test_for_selection=False, entities_subset=None, corrupt_side="s,o", focusE=False,
                              focusE_params={}, retrain_best_model=False, verbose=False):
    """Grid search (max_combinations=None) or random search (max_combinations=n, param_grid_random_seed) over the
    hyper-parameters of a ScoringBasedEmbeddingModel of scoring type model_class (protocol.py:447-932).

    param_grid: keys batch_size, epochs, k, eta, loss, loss_params, regularizer, regularizer_params, optimizer,
    optimizer_params, initializer, focusE_params, reciprocal_relations (extension: the constructor's flag, default
    False); values are lists, scalars, dicts of those, or callables (random search).  The caller's dict is not
    modified.  Candidates train with sampled corruptions, so one with reciprocal_relations=True is recorded with the
    model's refusal of that training.

    Each candidate is trained on X_train with early stopping on X_valid[::2] (EarlyStopping(monitor='val_<criteria>',
    mode='max', restore_best_weights=True); early_stopping_params: criteria 'mrr', burn_in 0, check_interval 10,
    stop_interval 5, validation_batch_size 10) and ranked on the selection set X_valid[1::2] (X_test with
    use_test_for_selection), filtered against {train, valid, test} with use_filter.  A candidate that raises is recorded
    as {"exception": str(e)}.  The best candidate by MRR (optionally retrained on X_train and X_valid[::2] for its
    early-stopping epoch count) is ranked on X_test.

    Returns (best_model, best_params, best_mrr_train, ranks_test, test_evaluation, experimental_history), as the
    reference's code does: test_evaluation is a dict of mrr, mr, hits_1, hits_3 and hits_10 (NaN without a model).
    verbose: progress lines on stdout and exceptions logged."""
    from .latent_features import EarlyStopping
    early_stopping_params = early_stopping_params or {}
    combinations, n_comb = _combinations(model_class, param_grid, max_combinations, param_grid_random_seed)
    callbacks = []
    if early_stopping:
        callbacks = [EarlyStopping(monitor="val_{}".format(early_stopping_params.get("criteria", "mrr")), min_delta=0,
                                   patience=early_stopping_params.get("stop_interval", 5), mode="max",
                                   restore_best_weights=True, verbose=int(bool(verbose)))]
    if focusE:
        assert isinstance(X_train, np.ndarray) and X_train.shape[1] > 3, \
            "Weights are missing! Concatenate them to X_train in order to use FocusE!"
    X_filter = {"train": X_train, "valid": X_valid, "test": X_test} if use_filter else None
    if use_test_for_selection:
        selection = X_test
    else:  # half of the validation set selects, the other half stops early
        selection, X_valid = X_valid[1::2], X_valid[::2]
    best_mrr_train, best_model, best_params, history = 0, None, None, []
    if verbose:
        print("Model selection over at most %d combinations" % n_comb)
    for params in combinations:
        result = {"model_name": params.pop("model_name"), "model_params": params}
        try:
            model = _build_model(model_class, params, _as_int32(params.get("eta", 1)))
            h = model.fit(X_train, batch_size=params.get("batch_size", 1000), epochs=params.get("epochs", 100),
                          validation_data=X_valid, validation_freq=early_stopping_params.get("check_interval", 10),
                          validation_batch_size=early_stopping_params.get("validation_batch_size", 10),
                          validation_burn_in=early_stopping_params.get("burn_in", 0), validation_corrupt_side="s,o",
                          validation_filter=X_filter, callbacks=callbacks, focusE=focusE,
                          focusE_params=params.get("focusE_params", {}), verbose=verbose)
            ranks = model.evaluate(selection, use_filter=X_filter, entities_subset=entities_subset,
                                   corrupt_side=corrupt_side, verbose=verbose)
            result["results"] = _metrics(ranks)
            if verbose:
                print("%s %s: %s" % (model_class, params, result["results"]))
            if result["results"]["mrr"] > best_mrr_train:
                best_mrr_train, best_model, best_params = result["results"]["mrr"], model, params
                params["early_stopping_epoch"] = len(h.history["loss"])  # epochs actually trained
        except Exception as e:
            result["results"] = {"exception": str(e)}
            if verbose:
                logger.error("Exception occurred for parameters:{}".format(params))
                logger.error(str(e))
        history.append(result)
    if best_model is None:
        nan = {k: np.nan for k in ("mrr", "mr", "hits_1", "hits_3", "hits_10")}
        return None, None, best_mrr_train, [], nan, history
    if retrain_best_model:
        if focusE:
            assert isinstance(X_valid, np.ndarray) and X_valid.shape[1] > 3, \
                "Validation set is used as training data for retraining the best model, but weights are missing. " \
                "Concatenate them to X_valid!"
        best_model = _build_model(model_class, best_params, best_params.get("eta", 1))
        best_model.fit(np.concatenate((X_train, X_valid)), batch_size=best_params.get("batch_size", 1000),
                       epochs=best_params.get("early_stopping_epoch"), validation_data=None, focusE=focusE,
                       focusE_params=best_params.get("focusE_params", {}), verbose=verbose)
    ranks_test = best_model.evaluate(X_test, use_filter=X_filter, verbose=verbose, entities_subset=entities_subset,
                                     corrupt_side=corrupt_side)
    test_evaluation = _metrics(ranks_test)
    if verbose:
        print("Best model test results: %s, model: %s, params: %s" % (test_evaluation, model_class, best_params))
    return best_model, best_params, best_mrr_train, ranks_test, test_evaluation, history
