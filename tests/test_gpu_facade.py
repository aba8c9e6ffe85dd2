"""GPU tests of the reference-facing facade (ScoringBasedEmbeddingModel) against the oracle:
BASELINE.json configs[0] (TransE k=50 eta=2, 1k entities / 10 relations) end to end."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _kg(E, R, n, seed=1, labels=True):
    rng = np.random.default_rng(seed)
    t = np.unique(np.stack([rng.integers(0, E, n), rng.integers(0, R, n), rng.integers(0, E, n)], 1), axis=0)
    rng.shuffle(t)
    if not labels:
        return t
    return np.stack([np.char.add("e", t[:, 0].astype(str)), np.char.add("r", t[:, 1].astype(str)),
                     np.char.add("e", t[:, 2].astype(str))], 1)


def _fit_pair(model_name, k, eta, loss, X, batch_size, epochs, optimizer="adam", loss_params=None, opt_params=None):
    """fit the facade and replay the same batches/corruptions through the CPU restatement."""
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel, loss_functions
    from oracle import ref_step
    from ampligraph_b200.datasets import DataIndexer
    ix = DataIndexer(X)
    E, R = ix.get_entities_count(), ix.get_relations_count()
    K = k if model_name in ("TransE", "DistMult") else 2 * k
    rng = np.random.default_rng(0)
    ent0 = rng.uniform(-0.3, 0.3, (E, K)).astype(np.float32)
    rel0 = rng.uniform(-0.3, 0.3, (R, K)).astype(np.float32)
    inits = [ent0, rel0] if model_name != "RotatE" else [ent0, "glorot_uniform"]
    m = ScoringBasedEmbeddingModel(eta=eta, k=k, scoring_type=model_name, seed=7)
    from ampligraph_b200.latent_features import optimizers
    m.compile(optimizer=optimizers.get(optimizer, dict(opt_params or {})), loss=loss_functions.get(loss, loss_params or {}),
              entity_relation_initializer=inits)
    hist = m.fit(X, batch_size=batch_size, epochs=epochs, verbose=False)
    # replay
    t = ix.get_indexes(X)
    if model_name == "RotatE":  # relations came from the engine's Glorot stream; rebuild the same start
        from ampligraph_b200.engine import KGEEngine
        e2 = KGEEngine(model_name, k, eta, E, R)
        e2.init_glorot_uniform(7)
        rel0 = e2.get_embeddings()[1].cpu().numpy()
        e2.close()
    rs = ref_step.RefStep(model_name, K, ent0, rel0, eta, loss=loss, loss_params=loss_params or {}, optimizer=optimizer,
                          optimizer_params=dict(opt_params or {}))
    step, losses = 0, []
    for _ in range(epochs):
        for s in range(0, len(t), batch_size):
            b = np.ascontiguousarray(t[s:s + batch_size])
            corr = m.engine.generate_corruptions(torch.as_tensor(b).cuda(), seed=7, step=step).cpu().numpy()
            losses.append(rs.train_step(b, corr))
            step += 1
    return m, rs, hist, losses, ix


def test_cfg1_transe_fit_predict_evaluate():
    """configs[0]: TransE k=50 eta=2 on a 1k-entity / 10-relation synthetic KG."""
    from oracle import c_oracle
    X = _kg(1000, 10, 10000)
    m, rs, hist, losses, ix = _fit_pair("TransE", 50, 2, "pairwise", X, batch_size=1000, epochs=3)
    # the logged loss is the never-reset running mean of per-batch SUM losses
    assert abs(hist.history["loss"][-1] - np.mean(losses)) <= 2e-4 * abs(np.mean(losses))
    ent = m.get_embeddings(ix.ent_labels, "e")
    rel = m.get_embeddings(ix.rel_labels, "r")
    assert ent.shape == (ix.get_entities_count(), 50)
    assert np.allclose(ent, rs.ent.detach().numpy(), rtol=1e-3, atol=2e-5)
    assert np.allclose(rel, rs.rel.detach().numpy(), rtol=1e-3, atol=2e-5)
    # predict == oracle scores on the SAME (GPU-trained) tables; unknown labels are dropped
    Xt = X[:200]
    sc = m.predict(np.concatenate([Xt, np.array([["nope", "r0", "e1"]])]))
    assert sc.shape == (200,)
    import exact_oracle as xo
    ratio = xo.PredictBound("TransE", ent, rel, ix.get_indexes(Xt)).assert_within(sc, "predict")
    print("\npredict: worst error / bound %.4f" % ratio)
    # evaluate: filtered ranks bit-exact against the oracle (+1, ScoringBasedEmbeddingModel.py:1684)
    test = X[:150]
    ranks = m.evaluate(test, use_filter={"train": X}, corrupt_side="s,o", verbose=False)
    assert ranks.shape == (150, 2) and ranks.dtype == np.int32
    tt, full = ix.get_indexes(test), ix.get_indexes(X)
    for j, (side, a, b, c) in enumerate((("s", 1, 2, 0), ("o", 0, 1, 2))):
        filt = [sorted(set(full[(full[:, a] == q[a]) & (full[:, b] == q[b])][:, c].tolist())) for q in tt]
        ref = c_oracle.rank_triples("TransE", side, "worst", ent, rel, tt, filters=filt)
        assert (ranks[:, j] == ref + 1).all()
    # MR('s,o') equals MR over separate 's' and 'o' runs (tests/ampligraph/evaluation/test_evaluate.py:66,:129)
    rs_ = m.evaluate(test, use_filter={"train": X}, corrupt_side="s", verbose=False)
    ro_ = m.evaluate(test, use_filter={"train": X}, corrupt_side="o", verbose=False)
    assert (rs_[:, 0] == ranks[:, 0]).all() and (ro_[:, 0] == ranks[:, 1]).all()
    rso = m.evaluate(test, use_filter={"train": X}, corrupt_side="s+o", verbose=False)
    assert (rso[:, 0] == ranks.sum(1) - 1).all()  # counts summed BEFORE the +1
    # entities_subset
    subset = ix.ent_labels[::7]
    rsub = m.evaluate(test, corrupt_side="o", entities_subset=subset, verbose=False)
    ref = c_oracle.rank_triples("TransE", "o", "worst", ent, rel, tt, cand_ids=ix.get_indexes(subset, "e"))
    assert (rsub[:, 0] == ref + 1).all()


@pytest.mark.parametrize("model_name,loss,optimizer", [("ComplEx", "self_adversarial", "adam"),
                                                       ("DistMult", "multiclass_nll", "adagrad"),
                                                       ("RotatE", "nll", "sgd"), ("HolE", "absolute_margin", "adam")])
def test_fit_tracks_oracle(model_name, loss, optimizer):
    X = _kg(300, 6, 3000, seed=3)
    # RotatE: phase = theta * pi/range (x17.8 here) makes the sum-over-batch SGD trajectory chaotic at the
    # default lr; a small lr keeps the two fp32 evaluations on the same trajectory
    opt_params = {"learning_rate": 1e-5} if model_name == "RotatE" else None
    m, rs, hist, losses, ix = _fit_pair(model_name, 16, 4, loss, X, batch_size=700, epochs=2, optimizer=optimizer,
                                        opt_params=opt_params)
    assert abs(hist.history["loss"][-1] - np.mean(losses)) <= 5e-4 * abs(np.mean(losses))
    ent = m.get_embeddings(ix.ent_labels, "e")
    assert np.allclose(ent, rs.ent.detach().numpy(), rtol=2e-3, atol=5e-5), np.abs(ent - rs.ent.detach().numpy()).max()


def test_user_callable_loss_and_validation_and_weights(tmp_path):
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    X = _kg(200, 5, 2000, seed=5)

    def user_loss(scores_pos, scores_neg):  # torch tensors instead of the reference's TF tensors
        return torch.nn.functional.softplus(1.0 - scores_pos + scores_neg).sum(0)

    m = ScoringBasedEmbeddingModel(eta=3, k=8, scoring_type="DistMult", seed=1)
    m.compile(optimizer="adam", loss=user_loss)
    h = m.fit(X[:1800], batch_size=600, epochs=4, validation_data=X[1800:], validation_freq=2, verbose=False)
    assert h.history["loss"][-1] < h.history["loss"][0]
    assert len(h.history["val_mrr"]) == 2 and 0 < h.history["val_mrr"][-1] <= 1
    p = str(tmp_path / "w.pkl")
    m.save_weights(p)
    m2 = ScoringBasedEmbeddingModel(eta=3, k=8, scoring_type="DistMult", seed=1)
    m2.compile(optimizer="adam", loss=user_loss)
    m2.load_weights(p)
    assert np.array_equal(m.predict(X[:50]), m2.predict(X[:50]))
    assert (m.evaluate(X[:20], verbose=False) == m2.evaluate(X[:20], verbose=False)).all()


@pytest.mark.parametrize("non_linearity", ["linear", "tanh", "softplus"])
def test_focuse_matches_oracle(non_linearity):
    """FocusE (ScoringBasedEmbeddingModel.py:342-368, :396-406): numeric edge values re-weight the
    scores before the loss; replayed with the oracle's scoring/loss restatements + autograd."""
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel, loss_functions
    from ampligraph_b200.datasets import DataIndexer
    from oracle import ref_step
    rng = np.random.default_rng(9)
    X = _kg(150, 4, 1200, seed=9)
    vals = rng.uniform(0, 1, (len(X), 1)).round(3)
    X4 = np.concatenate([X.astype(object), vals.astype(object)], axis=1)
    ix = DataIndexer(X)
    E, R, k, eta, bs = ix.get_entities_count(), ix.get_relations_count(), 10, 3, 500
    ent0 = rng.uniform(-0.3, 0.3, (E, k)).astype(np.float32)
    rel0 = rng.uniform(-0.3, 0.3, (R, k)).astype(np.float32)
    m = ScoringBasedEmbeddingModel(eta=eta, k=k, scoring_type="DistMult", seed=3)
    m.compile(optimizer="adam", loss=loss_functions.get("nll"), entity_relation_initializer=[ent0, rel0])
    params = {"non_linearity": non_linearity, "stop_epoch": 3, "structural_wt": 0.001}
    m.fit(X4, batch_size=bs, epochs=2, verbose=False, focusE=True, focusE_params=params)
    # replay on the CPU
    rs = ref_step.RefStep("DistMult", k, ent0, rel0, eta, loss="nll", optimizer="adam")
    nl = {"linear": lambda x: x, "tanh": torch.tanh,
          "softplus": lambda x: torch.log(1 + 9999 * torch.exp(x))}[non_linearity]
    t = ix.get_indexes(X)
    step = 0
    for epoch in range(2):
        sw = max(1 - epoch / 3, 0.001)
        for s0 in range(0, len(t), bs):
            b = np.ascontiguousarray(t[s0:s0 + bs])
            w = torch.tensor(vals[s0:s0 + bs, 0], dtype=torch.float32)
            corr = m.engine.generate_corruptions(torch.as_tensor(b).cuda(), seed=3, step=step).cpu().numpy()
            for v in (rs.ent, rs.rel):
                v.grad = None
            sp, sn = rs.forward(b, corr)
            fp = nl(sp) * (sw + (1 - sw) * (1 - w))
            fn = nl(sn) * (sw + (1 - sw) * w.repeat(eta))
            ref_step.total_loss("nll", fp, fn, eta).backward()
            with torch.no_grad():
                rs.opt.step({"ent": (rs.ent, rs.ent.grad), "rel": (rs.rel, rs.rel.grad)})
            step += 1
    ent = m.get_embeddings(ix.ent_labels, "e")
    assert np.allclose(ent, rs.ent.detach().numpy(), rtol=2e-3, atol=5e-5), np.abs(ent - rs.ent.detach().numpy()).max()


def test_calibration_and_early_stopping():
    """calibrate / predict_proba (ScoringBasedEmbeddingModel.py:1922-2212) and an EarlyStopping callback."""
    from ampligraph_b200.latent_features import EarlyStopping, ScoringBasedEmbeddingModel
    X = _kg(200, 5, 3000, seed=11)
    m = ScoringBasedEmbeddingModel(eta=5, k=16, scoring_type="ComplEx", seed=2)
    m.compile(optimizer="adam", loss="multiclass_nll")
    es = EarlyStopping(monitor="val_mrr", patience=1)
    h = m.fit(X[:2600], batch_size=650, epochs=60, validation_data=X[2600:], validation_freq=2, callbacks=[es], verbose=False)
    assert es.stopped_epoch is not None and len(h.history["loss"]) < 60  # stopped early
    with pytest.raises(RuntimeError):
        m.predict_proba(X[:10])
    rng = np.random.default_rng(0)
    X_neg = X[2600:].copy()
    X_neg[:, 2] = rng.permutation(X_neg[:, 2])  # corrupted objects
    m.calibrate(X[2600:], X_neg=X_neg, batch_size=100, epochs=30)
    p_pos, p_neg = m.predict_proba(X[2600:]), m.predict_proba(X_neg)
    assert ((p_pos > 0) & (p_pos < 1)).all() and p_pos.mean() > p_neg.mean()
    sc = m.predict(X[2600:])
    order = np.argsort(sc)
    assert (np.diff(p_pos[order]) >= -1e-7).all() or (np.diff(p_pos[order]) <= 1e-7).all()  # monotone in the score
    m.calibrate(X[2600:], positive_base_rate=0.5, batch_size=100, epochs=5)  # corruption-based variant
    assert m.is_calibrated and 0 < m.predict_proba(X[:5]).min()
    with pytest.raises(ValueError):
        m.calibrate(X[2600:], positive_base_rate=1.5)


def test_train_on_batches_equals_train_on_batch():
    """The streamed host path (copy-stream prefetch, loss read one step late) is the same sequence of train_steps as
    calling train_on_batch per batch: identical tables, identical per-batch losses; pinned and pageable sources."""
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel
    E, R, B = 300, 5, 256
    t = _kg(E, R, 3000, labels=False).astype(np.int32)
    batches = [np.ascontiguousarray(t[i:i + B]) for i in range(0, 5 * B, B)] + [np.ascontiguousarray(t[5 * B:5 * B + 100])]  # short last batch
    out = []
    for streamed in (False, True, "pinned"):
        m = ScoringBasedEmbeddingModel(eta=4, k=16, scoring_type="ComplEx", seed=3, max_ent_size=E, max_rel_size=R)
        m.data_indexer = False
        m.compile(optimizer="adam", loss="self_adversarial")
        if streamed is False:
            losses = [m.train_on_batch(torch.as_tensor(b)) for b in batches]
        elif streamed is True:
            losses = m.train_on_batches(iter(batches))
        else:
            losses = m.train_on_batches([torch.as_tensor(b).pin_memory() for b in batches], prefetch=3)
        out.append((losses, [x.cpu().numpy() for x in m.engine.get_embeddings()]))
    for losses, (e, r) in out[1:]:
        assert np.allclose(losses, out[0][0], rtol=1e-6) and len(losses) == len(batches)
        # same steps, but fp32 atomics (red.v4) sum in a different order from run to run: equal to rounding, not bit for bit
        assert np.allclose(e, out[0][1][0], rtol=1e-5, atol=1e-7) and np.allclose(r, out[0][1][1], rtol=1e-5, atol=1e-7)


def test_model_initializers_and_regularizer_pair():
    """compile() takes the Keras initialiser names / a pair, and a pair of regularisers (EmbeddingLookupLayer.py:105-155);
    the reference's own initialiser test: RandomNormal(mean=0.5, stddev=0.05) -> mean/std of the built tables."""
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel, initializers
    X = _kg(500, 6, 4000)
    m = ScoringBasedEmbeddingModel(eta=2, k=40, scoring_type="DistMult", seed=11)
    m.compile(optimizer="sgd", loss="nll", entity_relation_initializer=[initializers.RandomNormal(mean=0.5, stddev=0.05), "he_uniform"],
              entity_relation_regularizer=["l2", "l1_l2"])
    m.fit(X, batch_size=1000, epochs=0, verbose=False)  # builds the tables, trains nothing
    m.is_fitted = True
    ent = m.get_embeddings(m.data_indexer.ent_labels, "e")
    rel = m.get_embeddings(m.data_indexer.rel_labels, "r")
    assert abs(ent.mean() - 0.5) < 5e-3 and abs(ent.std() - 0.05) < 5e-3  # test_initializers.py:48-49
    lim = np.sqrt(6.0 / len(rel))
    assert np.abs(rel).max() <= lim and np.abs(rel).max() > 0.9 * lim
    h = m.fit(X, batch_size=1000, epochs=2, verbose=False)
    assert np.isfinite(h.history["loss"]).all()
