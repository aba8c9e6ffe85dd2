"""GPU tests of the evaluation protocol: select_best_model_ranking, fit(validation_split=...),
EarlyStopping(restore_best_weights=True) on both parameter-block paths, and the filter fit builds once for its
validations."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _kg(E=200, R=5, n=3000, seed=11):
    rng = np.random.default_rng(seed)
    t = np.unique(np.stack([rng.integers(0, E, n), rng.integers(0, R, n), rng.integers(0, E, n)], 1), axis=0)
    rng.shuffle(t)
    return np.stack([np.char.add("e", t[:, 0].astype(str)), np.char.add("r", t[:, 1].astype(str)),
                     np.char.add("e", t[:, 2].astype(str))], 1)


def _splits():
    from ampligraph_b200.evaluation import train_test_split_no_unseen
    X = _kg()
    rest, X_test = train_test_split_no_unseen(X, test_size=200, seed=0)
    X_train, X_valid = train_test_split_no_unseen(rest, test_size=200, seed=1)
    return X_train, X_valid, X_test


def _model(scoring="ComplEx", eta=2, k=16, lr=0.01, seed=0):
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel, optimizers
    m = ScoringBasedEmbeddingModel(eta=eta, k=k, scoring_type=scoring, seed=seed)
    m.compile(optimizer=optimizers.get("adam", {"learning_rate": lr}), loss="multiclass_nll")
    return m


def _check_result(out, n_test, n_candidates):
    best_model, best_params, best_mrr, ranks_test, test_eval, history = out
    assert len(history) == n_candidates
    mrrs = [h["results"]["mrr"] for h in history if "mrr" in h["results"]]
    assert mrrs and best_mrr == max(mrrs) and best_model is not None
    assert best_params["early_stopping_epoch"] >= 1
    assert np.asarray(ranks_test).shape == (n_test, 2)
    assert sorted(test_eval) == ["hits_1", "hits_10", "hits_3", "mr", "mrr"]
    assert all("model_name" not in h["model_params"] and "model_name" in h for h in history)
    return history


def test_select_best_model_ranking_grid():
    """Grid search: every combination tried in grid order; a candidate that raises is recorded, not fatal; Python
    ints as eta are accepted."""
    from ampligraph_b200.evaluation import mrr_score, select_best_model_ranking
    X_train, X_valid, X_test = _splits()
    grid = {"batch_size": [600], "epochs": [6], "k": [8, 16], "eta": 2, "loss": ["multiclass_nll", "no_such_loss"],
            "optimizer_params": {"learning_rate": [0.01]}}
    out = select_best_model_ranking("ComplEx", X_train, X_valid, X_test, grid,
                                    early_stopping_params={"check_interval": 2, "stop_interval": 1})
    history = _check_result(out, len(X_test), 4)
    assert "model_name" not in grid and grid["eta"] == 2  # the caller's grid is not modified
    assert [(h["model_params"]["k"], h["model_params"]["loss"]) for h in history] == \
        [(8, "multiclass_nll"), (8, "no_such_loss"), (16, "multiclass_nll"), (16, "no_such_loss")]
    assert [("exception" in h["results"]) for h in history] == [False, True, False, True]
    assert "no_such_loss" in history[1]["results"]["exception"]
    best_model, _, _, ranks_test, test_eval, _ = out
    assert test_eval["mrr"] == mrr_score(ranks_test)
    # the test ranks are the best model's filtered ranks of X_test
    again = best_model.evaluate(X_test, use_filter={"train": X_train, "valid": X_valid, "test": X_test})
    assert np.array_equal(again, ranks_test)


def test_select_best_model_ranking_random_retrain():
    """Random search with a callable, no early stopping, retrain of the best model on train + half of valid for its
    epoch count."""
    from ampligraph_b200.evaluation import select_best_model_ranking
    X_train, X_valid, X_test = _splits()
    grid = {"batch_size": [600], "epochs": [3, 4], "k": [8, 16], "eta": [2, 3],
            "optimizer_params": {"learning_rate": lambda: np.random.uniform(0.005, 0.02)}}
    state = np.random.get_state()
    out = select_best_model_ranking("DistMult", X_train, X_valid, X_test, grid, max_combinations=3,
                                    param_grid_random_seed=5, early_stopping=False, retrain_best_model=True,
                                    use_filter=False)
    assert all(np.array_equal(a, b) for a, b in zip(state, np.random.get_state()))
    history = _check_result(out, len(X_test), 3)
    best_model, best_params = out[0], out[1]
    assert all(isinstance(h["model_params"]["eta"], np.int32) for h in history)
    assert best_params["early_stopping_epoch"] == best_params["epochs"]  # no early stopping: every epoch ran
    assert all(h["results"].get("mrr") is not None for h in history)
    # retrained on X_train and X_valid[::2] for early_stopping_epoch epochs
    n = len(X_train) + len(X_valid[::2])
    assert len(best_model.history.history["loss"]) == best_params["early_stopping_epoch"]
    assert best_model._step == best_params["early_stopping_epoch"] * -(-n // 600)


def test_fit_validation_split_equals_manual_split():
    """fit(validation_split=f) trains on, and validates against, train_test_split_no_unseen(x, f, seed=model.seed)."""
    from ampligraph_b200.evaluation import train_test_split_no_unseen
    X = _kg()
    a = _model(seed=3)
    ha = a.fit(X, batch_size=500, epochs=3, validation_split=0.1, validation_freq=1, verbose=False)
    tr, va = train_test_split_no_unseen(X, test_size=0.1, seed=3)
    b = _model(seed=3)
    hb = b.fit(tr, batch_size=500, epochs=3, validation_data=va, validation_freq=1, verbose=False)
    # the same training rows in the same order: the indexer's first-seen order and the step count are those of tr
    assert list(a.data_indexer.ent_labels) == list(b.data_indexer.ent_labels) and a._step == b._step == 3 * 6
    # same steps, but the replaced rows' gradient sum is fp32 atomics whose order varies from run to run (see
    # test_train_on_batches_equals_train_on_batch): the tables agree to rounding, not bit for bit
    for x, y in zip(a.engine.get_embeddings(), b.engine.get_embeddings()):
        assert np.allclose(x.cpu().numpy(), y.cpu().numpy(), rtol=1e-4, atol=1e-6)
    assert np.allclose(ha.history["loss"], hb.history["loss"], rtol=1e-5)
    assert np.allclose(ha.history["val_mr"], hb.history["val_mr"], rtol=2e-2) and len(ha.history["val_mrr"]) == 3


class _Recorder:
    """Copies of the tables and the first slot at the end of every epoch (runs before EarlyStopping)."""

    def __init__(self):
        self.tables, self.slots = [], []

    def on_epoch_end(self, epoch, logs):
        eng = self.model.engine
        self.tables.append((eng.ent.clone(), eng.rel.clone()))
        self.slots.append(eng.slots["ent"][0].clone())


@pytest.mark.parametrize("batch_size,deferred", [(600, True), (20, False)])
def test_early_stopping_restores_best_tables(batch_size, deferred):
    """After the stop the tables are the best epoch's, bit for bit, whichever of the deferred steps' two parameter
    blocks is live; the optimizer slots are not restored.  The same instance then serves a second fit afresh."""
    from ampligraph_b200.latent_features import EarlyStopping
    X = _kg()
    es = EarlyStopping(monitor="val_mrr", min_delta=1.0, patience=3, restore_best_weights=True)
    runs = []
    for seed in (0, 1):
        m, rec = _model(lr=0.05, seed=seed), _Recorder()
        h = m.fit(X[:2600], batch_size=batch_size, epochs=30, validation_data=X[2600:], validation_freq=1,
                  callbacks=[rec, es], verbose=False)
        assert (m.engine._pblock_next is not None) == deferred  # which parameter-block path the steps took
        # min_delta=1: only the first validation improves, so the stop comes at epoch 3 and restores epoch 0
        assert es.model is m and es.stopped_epoch == 3 and es.best_epoch == 0 and len(h.history["loss"]) == 4
        assert not torch.equal(rec.tables[3][0], rec.tables[0][0])
        assert torch.equal(m.engine.ent, rec.tables[0][0]) and torch.equal(m.engine.rel, rec.tables[0][1])
        assert torch.equal(m.engine.slots["ent"][0], rec.slots[3])
        runs.append(m.predict(X[2600:2700]))
    assert not np.array_equal(runs[0], runs[1])


def test_early_stopping_best_epoch_by_mrr():
    """Without min_delta: the restored tables are those of the epoch with the highest val_mrr before the stop."""
    from ampligraph_b200.latent_features import EarlyStopping
    X = _kg()
    es = EarlyStopping(monitor="val_mrr", patience=2, restore_best_weights=True)
    m, rec = _model(lr=0.2, seed=4), _Recorder()
    h = m.fit(X[:2600], batch_size=600, epochs=60, validation_data=X[2600:], validation_freq=1, callbacks=[rec, es],
              verbose=False)
    mrr = h.history["val_mrr"]
    best = int(np.argmax(mrr))
    assert es.best_epoch == best and es.best == mrr[best]
    if es.stopped_epoch is not None:
        assert es.stopped_epoch == best + 2
        assert torch.equal(m.engine.ent, rec.tables[best][0]) and torch.equal(m.engine.rel, rec.tables[best][1])


def test_validation_filter_built_once_gives_same_ranks():
    """The FilterIndex fit builds once for its validations ranks exactly as evaluate(use_filter=dict) does."""
    X_train, X_valid, X_test = _splits()
    filt = {"train": X_train, "valid": X_valid, "test": X_test}
    m = _model()
    h = m.fit(X_train, batch_size=600, epochs=4, validation_data=X_valid, validation_freq=2, validation_filter=filt,
              verbose=False)
    for use_filter in (filt, True):
        fresh = m.evaluate(X_valid, use_filter=use_filter, verbose=False)
        kept = m._build_filter(use_filter, lambda: m._index(X_valid))
        assert np.array_equal(m.evaluate(X_valid, use_filter=use_filter, verbose=False, _filter_index=kept), fresh)
    from ampligraph_b200.evaluation import mrr_score
    assert h.history["val_mrr"][-1] == mrr_score(m.evaluate(X_valid, use_filter=filt, batch_size=10, verbose=False))
    raw = m.evaluate(X_valid, use_filter=False, verbose=False)
    assert not np.array_equal(raw, m.evaluate(X_valid, use_filter=filt, verbose=False))  # the filter mattered
