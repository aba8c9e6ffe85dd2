"""RMSprop, Adadelta and Adamax on the GPU: full training steps against the restatement of tests/optim_oracle.py, every
optimizer path (dense, deferred owner-per-row, lazy, sharded, exchange, data-parallel at world 1) against the others,
torch.optim as an independent check, the old config layout, the refusals and the facade's per-table semantics."""
import ctypes as C

import numpy as np
import pytest
import torch

import optim_oracle
from ampligraph_b200 import _lib
from ampligraph_b200.parallel import tables_close

pytestmark = pytest.mark.gpu

# (name, hyper-parameters): every kind and variant
VARIANTS = {
    "rmsprop": ("rmsprop", {"learning_rate": 0.01}),
    "rmsprop_centered": ("rmsprop", {"learning_rate": 0.01, "rho": 0.8, "centered": True}),
    "rmsprop_momentum": ("rmsprop", {"learning_rate": 0.01, "momentum": 0.9}),
    "adadelta": ("adadelta", {"learning_rate": 1.0}),
    "adamax": ("adamax", {"learning_rate": 0.01}),
}


def _engine(*a, **kw):
    from ampligraph_b200.engine import KGEEngine
    return KGEEngine(*a, **kw)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _dev(a):
    return torch.as_tensor(a).cuda().contiguous()


def _tables(model, E, R, k, rng, scale=0.5):
    K = k if model in ("TransE", "DistMult") else 2 * k
    return rng.uniform(-scale, scale, (E, K)).astype(np.float32), rng.uniform(-scale, scale, (R, K)).astype(np.float32)


def _triples(E, R, n, rng):
    return np.stack([rng.integers(0, E, n), rng.integers(0, R, n), rng.integers(0, E, n)], 1).astype(np.int32)


def _negatives(E, B, eta, rng):
    return rng.integers(0, E, B * eta).astype(np.int32), rng.integers(0, 2, B * eta).astype(np.uint8)


def _corruptions(t, neg_ent, neg_keep, eta):
    from oracle import c_oracle
    return c_oracle.corrupt(t, eta, neg_keep, neg_ent)


def _close(a, b, rtol):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b).max() <= rtol * max(np.abs(b).max(), 1e-30) + 1e-7


def _pads_zero(eng, k):
    blk = eng._pblock
    return bool((blk[:, k:eng.kp] == 0).all()) and (eng.ld == eng.kp or bool((blk[:, eng.kp + k:] == 0).all()))


def _bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


@pytest.mark.parametrize("reg", [None, {"p": 2, "lambda": 1e-3}, {"p": 3, "lambda": 1e-2}])
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_train_steps_vs_oracle(variant, reg):
    """Five full steps (fused kernel, deferred owner-per-row optimizer) track the restatement; k = 10 leaves pad columns,
    which stay exactly 0."""
    name, params = VARIANTS[variant]
    rng = np.random.default_rng(17)
    model, E, R, k, eta, B = "ComplEx", 50, 4, 10, 3, 40
    ent, rel = _tables(model, E, R, k, rng)
    eng = _engine(model, k, eta, E, R, loss="multiclass_nll", optimizer=name, optimizer_params=params, regularizer=reg)
    eng.set_embeddings(ent, rel)
    rs = optim_oracle.RefStep(model, 2 * k, ent, rel, eta, "multiclass_nll", {}, optimizer=name, optimizer_params=dict(params),
                              regularizer=({"p": reg["p"], "lam": reg["lambda"]} if reg else None))
    for step in range(5):
        t = _triples(E, R, B, rng)
        neg_ent, neg_keep = _negatives(E, B, eta, rng)
        eng.train_step(_dev(t), (_dev(neg_ent), _dev(neg_keep)))
        ref_loss = rs.train_step(t, _corruptions(t, neg_ent, neg_keep, eta))
        got_loss = eng.read_loss()
        assert abs(got_loss - ref_loss) <= 2e-4 * abs(ref_loss), (step, got_loss, ref_loss)
    got_ent, got_rel = (x.cpu().numpy() for x in eng.get_embeddings())
    assert _close(got_ent, rs.ent.detach().numpy(), 5e-4)
    assert _close(got_rel, rs.rel.detach().numpy(), 5e-4)
    assert _pads_zero(eng, k)
    eng.close()


def _zipf_triples(E, R, n, rng):
    w = 1.0 / np.arange(1, E + 1)
    cdf = np.cumsum(w / w.sum())
    perm = rng.permutation(E)
    s, o = perm[np.searchsorted(cdf, rng.random(n))], perm[np.searchsorted(cdf, rng.random(n))]
    return np.stack([s, rng.integers(0, R, n), o], 1).astype(np.int32)


@pytest.mark.parametrize("reg", [None, {"p": 2, "lambda": 1e-3}])
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_deferred_vs_plain(variant, reg):
    """The owner-per-row kernel (deferred steps) against the bucket sum + kge_optimizer_step on the same inputs."""
    name, params = VARIANTS[variant]
    E, R, B, k, eta = 500, 9, 1000, 30, 5
    t = _dev(_zipf_triples(E, R, B, np.random.default_rng(21)))
    ent, rel = _tables("ComplEx", E, R, k, np.random.default_rng(5), 0.3)
    out = {}
    for defer in (True, False):
        eng = _engine("ComplEx", k, eta, E, R, loss="self_adversarial", optimizer=name, optimizer_params=params, regularizer=reg)
        eng.set_embeddings(ent, rel)
        for step in range(3):
            eng.forward_backward(t, None, seed=3, step=step, defer=defer)
            assert eng._deferred == defer
            eng.apply_gradients()
        out[defer] = [x.cpu().numpy() for x in eng.get_embeddings()] + [eng.read_loss()]
        assert _pads_zero(eng, k)
        eng.close()
    for got, want, init in zip(out[True][:2], out[False][:2], (ent, rel)):
        ok, err = tables_close(got, want, init)
        assert ok, err
    assert abs(out[True][2] - out[False][2]) <= 1e-6 * abs(out[False][2])


@pytest.mark.parametrize("model,neg_group", [("DistMult", 0), ("ComplEx", 3)])
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_lazy_vs_restatement(variant, model, neg_group):
    """lazy_<name>: looked-up rows take the dense rule, other rows and their slots stay bit-unchanged.  Relation 0 is a
    zero row, so the entities of its triples are looked up with a gradient of exactly 0 in step 2: they are still
    updated (their slot 0 decays), as TensorFlow's IndexedSlices list them."""
    name, params = VARIANTS[variant]
    rng = np.random.default_rng(43)
    E, R, k, eta, B = 300, 4, 12, 3, 20
    ent, rel = _tables(model, E, R, k, rng)
    rel[0] = 0.0
    zero_rows = np.array([7, 8], np.int32)
    eng = _engine(model, k, eta, E, R, loss="nll", optimizer="lazy_" + name, optimizer_params=params, neg_group=neg_group)
    assert eng.lazy_tables == {"ent": True, "rel": True}
    eng.set_embeddings(ent, rel)
    rs = optim_oracle.RefStep(model, ent.shape[1], ent, rel, eta, "nll", {}, optimizer="lazy_" + name,
                              optimizer_params=dict(params))
    others = np.setdiff1d(np.arange(E), zero_rows)
    touched = np.zeros(E, bool)
    slot_after = {}
    for step in range(3):
        t = _triples(E, R, B, rng)
        t[:, 1] = rng.integers(1, R, B)
        t[:, [0, 2]] = rng.choice(others, (B, 2))
        if step == 0:
            t[:2, 0] = zero_rows  # a non-zero gradient first, so that the slots hold something to decay
        if step == 1:
            t[:2] = [[zero_rows[0], 0, zero_rows[1]], [zero_rows[1], 0, zero_rows[0]]]
        neg_ent, neg_keep = rng.choice(others, B * eta).astype(np.int32), rng.integers(0, 2, B * eta).astype(np.uint8)
        eng.train_step(_dev(t), (_dev(neg_ent), _dev(neg_keep)), step=step)
        rs.train_step(t, _corruptions(t, neg_ent, neg_keep, eta))
        touched[t[:, 0]] = touched[t[:, 2]] = touched[neg_ent] = True
        slot_after[step] = eng.slots["ent"][0][zero_rows].clone()
    # the zero-gradient rows were updated in step 2: every non-zero slot element decayed
    assert bool((slot_after[0] != 0).any()) and bool(((slot_after[1] != slot_after[0]) | (slot_after[0] == 0)).all())
    got_ent, got_rel = (x.cpu().numpy() for x in eng.get_embeddings())
    assert (got_ent[~touched] == ent[~touched]).all()
    assert (eng.slots["ent"][0][torch.as_tensor(~touched).cuda()] == 0).all()
    assert _close(got_ent, rs.ent.detach().numpy(), 5e-4)
    assert _close(got_rel, rs.rel.detach().numpy(), 5e-4)
    eng.close()


def _packed(rows, ld, k, rng, scale):
    x = np.zeros((rows, ld), np.float32)
    x[:, :k] = rng.uniform(-scale, scale, (rows, k))
    return x


def _slots(cfg, rows, ld):
    from ampligraph_b200.engine import optimizer_slots
    return [None if v is None else torch.full((max(rows, 1), ld), v, dtype=torch.float32, device="cuda")
            for v in optimizer_slots(cfg)]


def _rank_order_sum(gs):
    acc = gs[0].copy()
    for g in gs[1:]:
        acc = acc + g
    return acc


@pytest.mark.parametrize("W", [2, 3, 8])
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_sharded_and_exchange_bit_equal(variant, W):
    """kge_optimizer_step_sharded and kge_optimizer_step_exchange (phases 0) with W replicas on one GPU, rank r = 0..W-1
    in turn: replicas bit-identical and bit-equal to kge_optimizer_step on the fp32 rank-order sum, slot shards equal to
    the plain slots, and within 1e-5 of the restatement."""
    from ampligraph_b200.parallel import row_shard
    name, params = VARIANTS[variant]
    rng = np.random.default_rng(W * 101 + len(variant))
    E, R, k = 97, 7, 10
    blk = E + R
    eng = _engine("DistMult", k, 1, E, R, optimizer=name, optimizer_params=params,
                  regularizer=[{"p": 2, "lambda": 1e-3}, {"p": 3, "lambda": 2e-3}])
    ce, cr, ld, lib = eng.opt_cfgs["ent"], eng.opt_cfgs["rel"], eng.ld, eng.lib
    bounds = [row_shard(blk, W, r) for r in range(W)]
    x0 = _packed(blk, ld, k, rng, 0.5)
    ex, sh, plain = [_dev(x0) for _ in range(W)], [_dev(x0[E:]) for _ in range(W)], _dev(x0)
    ex_slots, pslots = [_slots(ce, hi - lo, ld) for lo, hi in bounds], _slots(ce, blk, ld)
    rb = [row_shard(R, W, r) for r in range(W)]
    sh_slots, rslots = [_slots(cr, hi - lo, ld) for lo, hi in rb], _slots(cr, R, ld)
    other = [torch.empty((blk, ld), device="cuda") for _ in range(W)]
    etp = (C.c_void_p * W)(*[x.data_ptr() for x in ex])
    stp = (C.c_void_p * W)(*[x.data_ptr() for x in sh])
    cut = lambda x, lo, hi: None if x is None else x[lo:hi]
    x_ref = torch.as_tensor(x0.copy())
    a_ref, b_ref = torch.zeros_like(x_ref), torch.zeros_like(x_ref)
    for t in (1, 2):
        gs = [_packed(blk, ld, k, rng, 1.0) for _ in range(W)]
        grads = [_dev(g) for g in gs]
        gp = (C.c_void_p * W)(*[g.data_ptr() for g in grads])
        rgp = (C.c_void_p * W)(*[g[E:].data_ptr() for g in grads])
        for r, (lo, hi) in enumerate(bounds):
            _lib.check(lib.kge_optimizer_step_exchange(eng.h, C.byref(ce), C.byref(cr), t, W, r, etp, gp, None, None,
                                                       _ptr(other[r]), _ptr(ex_slots[r][0]), _ptr(ex_slots[r][1]), lo, hi,
                                                       None, t, 0, None, eng._stream()))
        for r, (lo, hi) in enumerate(rb):
            _lib.check(lib.kge_optimizer_step_sharded(eng.h, C.byref(cr), t, W, r, stp, rgp, _ptr(sh_slots[r][0]),
                                                      _ptr(sh_slots[r][1]), lo, hi, None, eng._stream()))
        gsum = _rank_order_sum(gs)
        gsum_d = _dev(gsum)
        for cfg, lo, hi in ((ce, 0, E), (cr, E, blk)):
            _lib.check(lib.kge_optimizer_step(eng.h, C.byref(cfg), t, _ptr(plain[lo:hi]), _ptr(gsum_d[lo:hi]),
                                              _ptr(cut(pslots[0], lo, hi)), _ptr(cut(pslots[1], lo, hi)), hi - lo, None,
                                              eng._stream()))
        torch.cuda.synchronize()
        assert all(_bits_equal(x, plain) for x in ex)
        assert all(_bits_equal(x, plain[E:]) for x in sh)
        for j in (0, 1):
            if pslots[j] is not None:
                assert _bits_equal(torch.cat([ex_slots[r][j][:hi - lo] for r, (lo, hi) in enumerate(bounds)]), pslots[j])
                assert _bits_equal(torch.cat([sh_slots[r][j][:hi - lo] for r, (lo, hi) in enumerate(rb)]), pslots[j][E:])
        g_t = torch.as_tensor(gsum)
        reg_g = torch.cat([2e-3 * x_ref[:E], 3 * 2e-3 * x_ref[E:].abs() ** 2 * torch.sign(x_ref[E:])])
        optim_oracle.rule(name, x_ref, g_t + reg_g, a_ref, b_ref, t, params["learning_rate"], params)
        assert _close(plain.cpu().numpy(), x_ref.numpy(), 1e-5)
    eng.close()


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_data_parallel_world_1(variant):
    """DataParallelTrainer on one GPU (deferred steps) against forward_backward + apply_gradients."""
    from ampligraph_b200.parallel import DataParallelTrainer
    name, params = VARIANTS[variant]
    rng = np.random.default_rng(37)
    E, R, B, k, eta = 1500, 11, 2000, 40, 6
    t = _dev(_zipf_triples(E, R, B, rng))
    ent, rel = _tables("ComplEx", E, R, k, rng, 0.3)
    make = lambda alloc: _engine("ComplEx", k, eta, E, R, loss="self_adversarial", optimizer=name, optimizer_params=params,
                                 table_alloc=alloc)
    dp = DataParallelTrainer(make)
    assert dp.mode == "single"
    ref = make(None)
    for e in (dp.eng, ref):
        e.set_embeddings(ent, rel)
    for step in range(3):
        dp.train_step(t, None, seed=1, step=step)
        ref.forward_backward(t, None, seed=1, step=step)
        ref.apply_gradients()
    for got, want, init in zip(dp.eng.get_embeddings(), ref.get_embeddings(), (ent, rel)):
        ok, err = tables_close(got.cpu().numpy(), want.cpu().numpy(), init)
        assert ok, err
    dp.close()
    ref.close()


def _step_once(eng, cfg, table, grad, slots, t):
    _lib.check(eng.lib.kge_optimizer_step(eng.h, C.byref(cfg), t, _ptr(table), _ptr(grad), _ptr(slots[0]), _ptr(slots[1]),
                                          table.shape[0], None, eng._stream()))


@pytest.mark.parametrize("torch_opt,name,params", [
    ("RMSprop", "rmsprop", {"learning_rate": 0.01, "rho": 0.9}),
    ("RMSprop", "rmsprop", {"learning_rate": 0.01, "rho": 0.8, "centered": True}),
    ("Adadelta", "adadelta", {"learning_rate": 1.0, "rho": 0.95})])
def test_against_torch_optim(torch_opt, name, params):
    """An independent restatement: torch.optim.RMSprop (alpha = rho, momentum 0) and torch.optim.Adadelta, three steps."""
    rng = np.random.default_rng(3)
    rows, k = 64, 10
    eng = _engine("DistMult", k, 1, 8, rows, optimizer=name, optimizer_params=params)
    cfg, ld = eng.opt_cfgs["rel"], eng.ld
    x0 = _packed(rows, ld, k, rng, 0.5)
    table, slots = _dev(x0), _slots(cfg, rows, ld)
    p = torch.nn.Parameter(torch.as_tensor(x0[:, :k].astype(np.float64)))
    if torch_opt == "RMSprop":
        opt = torch.optim.RMSprop([p], lr=params["learning_rate"], alpha=params["rho"], eps=1e-7,
                                  centered=params.get("centered", False))
    else:
        opt = torch.optim.Adadelta([p], lr=params["learning_rate"], rho=params["rho"], eps=1e-7)
    for t in (1, 2, 3):
        g = _packed(rows, ld, k, rng, 1.0)
        _step_once(eng, cfg, table, _dev(g), slots, t)
        p.grad = torch.as_tensor(g[:, :k].astype(np.float64))
        opt.step()
    torch.cuda.synchronize()
    got = table.cpu().numpy()
    assert np.allclose(got[:, :k], p.detach().numpy(), rtol=1e-5, atol=1e-7)
    assert (got[:, k:] == 0).all()
    eng.close()


class _OldConfig(C.Structure):  # kge_optimizer_config as built against the header before rho / centered
    _fields_ = _lib.KgeOptimizerConfig._fields_[:12]


def test_old_config_layout():
    """A config of the old struct_size drives Adam bit-identically to the current layout; a new kind in it is refused
    and launches nothing."""
    rng = np.random.default_rng(11)
    rows, k = 40, 12
    eng = _engine("DistMult", k, 1, 8, rows, optimizer="adam", optimizer_params={"learning_rate": 0.01})
    new, ld = eng.opt_cfgs["rel"], eng.ld
    old = _OldConfig(C.sizeof(_OldConfig), *[getattr(new, f) for f, _ in _OldConfig._fields_[1:]])
    assert C.sizeof(_OldConfig) == 48
    x0 = _packed(rows, ld, k, rng, 0.5)
    ta, tb = _dev(x0), _dev(x0)
    sa, sb = _slots(new, rows, ld), _slots(new, rows, ld)
    for t in (1, 2):
        g = _packed(rows, ld, k, rng, 1.0)
        _step_once(eng, new, ta, _dev(g), sa, t)
        _lib.check(eng.lib.kge_optimizer_step(eng.h, C.cast(C.pointer(old), C.POINTER(_lib.KgeOptimizerConfig)), t, _ptr(tb),
                                              _ptr(_dev(g)), _ptr(sb[0]), _ptr(sb[1]), rows, None, eng._stream()))
    torch.cuda.synchronize()
    assert _bits_equal(ta, tb) and _bits_equal(sa[0], sb[0]) and _bits_equal(sa[1], sb[1])
    old.kind = _lib.OPTIMIZERS["adamax"]
    g = _dev(_packed(rows, ld, k, rng, 1.0))
    before = tb.clone()
    with pytest.raises(ValueError, match="optimizer identifier"):
        _lib.check(eng.lib.kge_optimizer_step(eng.h, C.cast(C.pointer(old), C.POINTER(_lib.KgeOptimizerConfig)), 3, _ptr(tb),
                                              _ptr(g), _ptr(sb[0]), _ptr(sb[1]), rows, None, eng._stream()))
    torch.cuda.synchronize()
    assert _bits_equal(tb, before) and bool((g != 0).any())
    eng.close()


def test_centered_rmsprop_with_momentum_refused():
    """Three slots would be needed: the library returns KGE_ERR_UNSUPPORTED and launches nothing (the gradient is not
    zeroed), the engine refuses to build such an optimizer."""
    rng = np.random.default_rng(13)
    rows, k = 16, 8
    eng = _engine("DistMult", k, 1, 8, rows, optimizer="rmsprop", optimizer_params={"centered": True})
    cfg, ld = eng.opt_cfgs["rel"], eng.ld
    cfg.momentum = 0.9
    table, grad = _dev(_packed(rows, ld, k, rng, 0.5)), _dev(_packed(rows, ld, k, rng, 1.0))
    t0, g0 = table.clone(), grad.clone()
    s = [torch.zeros_like(table), torch.zeros_like(table)]
    with pytest.raises(NotImplementedError):
        _step_once(eng, cfg, table, grad, s, 1)
    torch.cuda.synchronize()
    assert _bits_equal(table, t0) and _bits_equal(grad, g0) and not s[0].any() and not s[1].any()
    with pytest.raises(NotImplementedError):
        eng.set_optimizer("rmsprop", {"centered": True, "momentum": 0.5})
    eng.close()


def _kg(E, R, n, seed=1):
    rng = np.random.default_rng(seed)
    t = np.unique(np.stack([rng.integers(0, E, n), rng.integers(0, R, n), rng.integers(0, E, n)], 1), axis=0)
    rng.shuffle(t)
    return np.stack([np.char.add("e", t[:, 0].astype(str)), np.char.add("r", t[:, 1].astype(str)),
                     np.char.add("e", t[:, 2].astype(str))], 1)


@pytest.mark.parametrize("optimizer,params,lazy", [
    ("adamax", {"learning_rate": 0.01}, {"ent": False, "rel": True}),
    ("rmsprop", {"learning_rate": 0.01, "momentum": 0.5}, {"ent": False, "rel": True}),
    ("adadelta", {"learning_rate": 1.0}, {"ent": False, "rel": False})])
def test_facade_fit_per_table_semantics(optimizer, params, lazy, tmp_path):
    """compile + fit for two epochs with an L2 regulariser on the entities only: the entity table takes the dense rule,
    the relation table the reference's rule for its optimizer (looked-up rows for Adamax and RMSprop with momentum);
    then save_weights / load_weights restore the state and training resumes from it."""
    from ampligraph_b200.datasets import DataIndexer
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel, loss_functions, optimizers, regularizers
    X = _kg(200, 12, 2000, seed=3)
    ix = DataIndexer(X)
    E, R, k, eta, bs = ix.get_entities_count(), ix.get_relations_count(), 16, 3, 500
    rng = np.random.default_rng(0)
    ent0 = rng.uniform(-0.3, 0.3, (E, 2 * k)).astype(np.float32)
    rel0 = rng.uniform(-0.3, 0.3, (R, 2 * k)).astype(np.float32)
    lam = 1e-3

    def model():
        m = ScoringBasedEmbeddingModel(eta=eta, k=k, scoring_type="ComplEx", seed=7)
        m.compile(optimizer=optimizers.get(optimizer, dict(params)), loss=loss_functions.get("nll"),
                  entity_relation_initializer=[ent0, rel0],
                  entity_relation_regularizer=[regularizers.LP_regularizer({"p": 2, "lambda": lam}), None])
        return m

    m = model()
    m.fit(X, batch_size=bs, epochs=2, verbose=False)
    assert m.engine.lazy_tables == lazy
    rs = optim_oracle.RefStep("ComplEx", 2 * k, ent0, rel0, eta, "nll", {}, optimizer=optimizer,
                              optimizer_params=dict(params), regularizer=[{"p": 2, "lam": lam}, None], lazy_tables=lazy)
    t = ix.get_indexes(X)
    step = 0
    for _ in range(2):
        for s in range(0, len(t), bs):
            b = np.ascontiguousarray(t[s:s + bs])
            rs.train_step(b, m.engine.generate_corruptions(torch.as_tensor(b).cuda(), seed=7, step=step).cpu().numpy())
            step += 1
    got_ent, got_rel = (x.cpu().numpy() for x in m.engine.get_embeddings())
    assert np.allclose(got_ent, rs.ent.detach().numpy(), rtol=2e-3, atol=5e-5)
    assert np.allclose(got_rel, rs.rel.detach().numpy(), rtol=2e-3, atol=5e-5)
    # save / load restores tables and slots bit for bit; one more epoch from there tracks the run that kept going (the
    # training kernel sums gradient rows in no fixed order, so two runs agree to rounding, not bit for bit)
    path = str(tmp_path / "w.pkl")
    m.save_weights(path)
    saved = [x.clone() for x in m.engine.get_embeddings()]
    saved_slots = {key: [None if s_ is None else s_.clone() for s_ in v] for key, v in m.engine.slots.items()}
    m.fit(X, batch_size=bs, epochs=1, verbose=False)
    m2 = model()
    m2.load_weights(path)
    assert m2.engine.lazy_tables == lazy and m2.engine.t == step
    for a, b in zip(m2.engine.get_embeddings(), saved):
        assert _bits_equal(a, b)
    for key, v in saved_slots.items():
        for a, b in zip(m2.engine.slots[key], v):
            assert (a is None and b is None) or _bits_equal(a, b)
    m2.fit(X, batch_size=bs, epochs=1, verbose=False)
    for a, b, init in zip(m2.engine.get_embeddings(), m.engine.get_embeddings(), saved):
        ok, err = tables_close(a.cpu().numpy(), b.cpu().numpy(), init.cpu().numpy())
        assert ok, err


def test_lazy_relation_table_refused_under_replication():
    """An engine whose relation table alone is lazy counts as lazy for the replicated trainer's check, and it registers
    both stamp buffers (the kernels stamp only while the entity buffer is set)."""
    from ampligraph_b200.parallel import reject_lazy
    eng = _engine("ComplEx", 8, 2, 30, 4, optimizer="adamax", lazy_tables=(False, True))
    assert eng.lazy and eng.stamps["ent"] is not None and eng.stamps["rel"] is not None
    with pytest.raises(NotImplementedError):
        reject_lazy("lazy_" if eng.lazy else "", 2)
    eng.close()
