"""Deferred steps (KGE_STEP_FUSED_DEFER + kge_optimizer_step_deferred: the replaced-row sum and the dense optimizer in one
owner-per-row launch, double-buffered parameter block) against the same steps without defer on the same seeded inputs.
The fused kernel is the same, so the first step's scores are bit-equal; gradients differ only in the order of the fp32
additions, so tables, slots and losses agree to rounding."""
import ctypes as C

import numpy as np
import pytest
import torch

from ampligraph_b200 import _lib
from ampligraph_b200.parallel import tables_close

pytestmark = pytest.mark.gpu


def _engine(*a, **kw):
    from ampligraph_b200.engine import KGEEngine
    return KGEEngine(*a, **kw)


def _tables(model, E, R, k, rng, scale=0.3):
    K = k if model == "DistMult" else 2 * k
    return rng.uniform(-scale, scale, (E, K)).astype(np.float32), rng.uniform(-scale, scale, (R, K)).astype(np.float32)


def _zipf_triples(E, R, n, rng):
    w = 1.0 / np.arange(1, E + 1)
    cdf = np.cumsum(w / w.sum())
    perm = rng.permutation(E)
    s, o = perm[np.searchsorted(cdf, rng.random(n))], perm[np.searchsorted(cdf, rng.random(n))]
    return np.stack([s, rng.integers(0, R, n), o], 1).astype(np.int32)


def _dev(a):
    return torch.as_tensor(a).cuda().contiguous()


def _close(a, b, rtol):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b).max() <= rtol * max(np.abs(b).max(), 1e-30) + 1e-7


def _pads_zero(eng, k):
    blk = eng._pblock
    return bool((blk[:, k:eng.kp] == 0).all()) and (eng.ld == eng.kp or bool((blk[:, eng.kp + k:] == 0).all()))


def _run(defer, model, k, eta, E, R, t, negatives=None, steps=3, optimizer="adam", opt_params=None, regularizer=None,
         between=None):
    rng = np.random.default_rng(5)
    ent, rel = _tables(model, E, R, k, rng)
    eng = _engine(model, k, eta, E, R, loss="self_adversarial", optimizer=optimizer,
                  optimizer_params=opt_params or {"learning_rate": 1e-3}, regularizer=regularizer)
    eng.set_embeddings(ent, rel)
    B = t.shape[0]
    sp, sn = torch.empty(B, device="cuda"), torch.empty(eta * B, device="cuda")
    neg = tuple(_dev(x) for x in negatives) if negatives is not None else None
    losses, scores = [], None
    for step in range(steps):
        launches = eng.launches
        eng.forward_backward(_dev(t), neg, seed=3, step=step, scores_pos=sp, scores_neg=sn, defer=defer)
        assert eng._deferred == defer  # the deferred path ran where it was asked for
        eng.apply_gradients()
        # pre-pass (3), fused kernel, then the bucket sum and the optimizer: one launch deferred, two otherwise
        assert eng.launches - launches == (5 if defer else 6)
        if step == 0:
            scores = (sp.cpu().numpy().copy(), sn.cpu().numpy().copy())
        losses.append(eng.read_loss())
        if between is not None:
            between(eng, step)
    ent_after, rel_after = (x.cpu().numpy() for x in eng.get_embeddings())
    slots = [s.cpu().numpy() for s in eng._sblocks if s is not None]
    assert _pads_zero(eng, k)
    eng.close()
    return dict(scores=scores, losses=losses, ent=ent_after, rel=rel_after, slots=slots, init=(ent, rel))


def _compare(a, b, adam):
    assert (a["scores"][0] == b["scores"][0]).all() and (a["scores"][1] == b["scores"][1]).all()
    for la, lb in zip(a["losses"], b["losses"]):
        assert abs(la - lb) <= 1e-6 * abs(lb), (la, lb)
    for key, init in (("ent", b["init"][0]), ("rel", b["init"][1])):
        if adam:
            # Adam turns a rounding difference in a gradient that cancels to ~0 into a visible step of that element:
            # the update-relative criterion of the multi-GPU parity checks
            ok, err = tables_close(a[key], b[key], init)
            assert ok, (key, err)
        else:
            assert _close(a[key], b[key], 1e-5), key
    for sa, sb in zip(a["slots"], b["slots"]):
        assert _close(sa, sb, 1e-5)


def _both(*a, adam=None, **kw):
    d = _run(True, *a, **kw)
    n = _run(False, *a, **kw)
    _compare(d, n, kw.get("optimizer", "adam") == "adam" if adam is None else adam)
    return d, n


def test_deferred_cfg2_full_size():
    """bench.py's workload: ComplEx k=200, eta=10, 14,505 entities, 237 relations, 27,212 Zipf positives, Adam; three
    steps, so the final tables are in the second block."""
    rng = np.random.default_rng(13)
    E, R, B = 14505, 237, 27212
    _both("ComplEx", 200, 10, E, R, _zipf_triples(E, R, B, rng))


@pytest.mark.parametrize("optimizer,params", [("adam", None), ("sgd", None), ("sgd", {"learning_rate": 1e-3, "momentum": 0.9}),
                                              ("adagrad", None)])
@pytest.mark.parametrize("regularizer", [None, {"p": 2, "lambda": 1e-3}, {"p": 1, "lambda": 1e-3, "p2": 2, "lambda2": 1e-3}])
def test_deferred_optimizers_and_regularizers(optimizer, params, regularizer):
    rng = np.random.default_rng(21)
    E, R, B = 500, 9, 1000
    _both("ComplEx", 30, 5, E, R, _zipf_triples(E, R, B, rng), optimizer=optimizer, opt_params=params,
          regularizer=regularizer)


@pytest.mark.parametrize("model,k,eta,E,B", [("DistMult", 400, 20, 3000, 2000),  # cfg3's row width (NIT = 4)
                                             ("DistMult", 7, 3, 500, 1000), ("HolE", 50, 7, 900, 777),
                                             ("ComplEx", 30, 1, 300, 501), ("HolE", 13, 32, 400, 333)])
def test_deferred_shapes(model, k, eta, E, B):
    rng = np.random.default_rng(23)
    _both(model, k, eta, E, 9, _zipf_triples(E, 9, B, rng))


def test_deferred_empty_buckets():
    """Injected negatives replace only entities [0, 1000): the other half have empty buckets and, outside the positives,
    no gradient at all, but still take the dense update (here the L2 regulariser's pull)."""
    rng = np.random.default_rng(29)
    E, R, B, eta = 2000, 7, 400, 5
    t = _zipf_triples(1000, R, B, rng)
    neg = (rng.integers(0, 1000, B * eta).astype(np.int32), rng.integers(0, 2, B * eta).astype(np.uint8))
    d, _ = _both("ComplEx", 30, eta, E, R, t, neg, regularizer={"p": 2, "lambda": 1e-2})
    idle = np.setdiff1d(np.arange(1000, E), np.concatenate([t[:, 0], t[:, 2]]))
    assert idle.size > 0 and (d["ent"][idle] != d["init"][0][idle]).any(1).all()


@pytest.mark.parametrize("model,k,eta", [("ComplEx", 200, 10), ("DistMult", 33, 5)])
def test_deferred_skewed_injected_negatives(model, k, eta):
    """Every corruption replaces one of 3 entities: buckets of thousands of entries, each walked by its one owner warp."""
    rng = np.random.default_rng(17)
    E, R, B = 700, 7, 4000
    t = _zipf_triples(E, R, B, rng)
    neg = (rng.choice(np.array([3, 77, 500], np.int32), B * eta), rng.integers(0, 2, B * eta).astype(np.uint8))
    _both(model, k, eta, E, R, t, neg, steps=2)


def test_deferred_embeddings_between_steps():
    """get_embeddings / set_embeddings between deferred steps address the current block."""
    rng = np.random.default_rng(31)
    E, R, B = 600, 5, 1200
    seen = {}

    def between(eng, step):
        ent, rel = eng.get_embeddings()
        seen.setdefault(step, []).append(ent.cpu().numpy())
        if step == 0:
            eng.set_embeddings(0.5 * ent, rel)

    _both("ComplEx", 30, 5, E, R, _zipf_triples(E, R, B, rng), between=between)
    assert _close(seen[1][0], seen[1][1], 1e-5)


def test_deferred_data_parallel_world_1():
    """DataParallelTrainer on one GPU ('single') defers; the same steps through forward_backward + apply_gradients."""
    from ampligraph_b200.parallel import DataParallelTrainer
    rng = np.random.default_rng(37)
    E, R, B, k, eta = 1500, 11, 2000, 40, 6
    t = _dev(_zipf_triples(E, R, B, rng))
    ent, rel = _tables("ComplEx", E, R, k, rng)
    make = lambda alloc: _engine("ComplEx", k, eta, E, R, loss="self_adversarial", optimizer="adam", table_alloc=alloc)
    dp = DataParallelTrainer(make)
    assert dp.mode == "single"
    ref = make(None)
    for e in (dp.eng, ref):
        e.set_embeddings(ent, rel)
    for step in range(3):
        dp.train_step(t, None, seed=1, step=step)
        ref.forward_backward(t, None, seed=1, step=step)
        ref.apply_gradients()
    assert dp.eng._pblock_next is not None and ref._pblock_next is None  # only the trainer's steps were deferred
    for got, want, init in zip(dp.eng.get_embeddings(), ref.get_embeddings(), (ent, rel)):
        ok, err = tables_close(got.cpu().numpy(), want.cpu().numpy(), init)
        assert ok, err
    got, want = dp.eng.read_loss(), ref.read_loss()
    assert abs(got - want) <= 1e-6 * abs(want)
    dp.close()
    ref.close()


def test_deferred_sum_must_be_consumed():
    """kge_optimizer_step_deferred needs a pending step; a pending step blocks the next kge_train_step."""
    rng = np.random.default_rng(41)
    E, R, B = 300, 5, 400
    eng = _engine("ComplEx", 16, 4, E, R, optimizer="adam")
    eng.set_embeddings(*_tables("ComplEx", E, R, 16, rng))
    t = _dev(_zipf_triples(E, R, B, rng))
    other = torch.empty_like(eng._pblock)
    args = lambda: (eng.h, C.byref(eng.opt_cfg), 1, C.c_void_p(eng._pblock.data_ptr()), C.c_void_p(other.data_ptr()),
                    C.c_void_p(eng._gblock.data_ptr()), C.c_void_p(eng._sblocks[0].data_ptr()),
                    C.c_void_p(eng._sblocks[1].data_ptr()), E + R, None, eng._stream())
    with pytest.raises(ValueError, match="no deferred step"):
        _lib.check(eng.lib.kge_optimizer_step_deferred(*args()))
    eng.forward_backward(t, None, defer=True)
    assert eng._deferred
    with pytest.raises(ValueError, match="pending"):
        eng.forward_backward(t, None, step=1)
    # refused arguments launch nothing and leave the step pending, in the library and in the engine
    bad = list(args())
    bad[8] = E + R - 1
    with pytest.raises(ValueError, match="blocks"):
        _lib.check(eng.lib.kge_optimizer_step_deferred(*bad))
    eng.opt_cfgs["ent"].kind = 7
    with pytest.raises(ValueError):
        eng.apply_gradients()
    assert eng._deferred and eng.t == 0
    eng.opt_cfgs["ent"].kind = _lib.OPTIMIZERS["adam"]
    eng.apply_gradients()
    assert not eng._deferred and eng.t == 1
    eng.forward_backward(t, None, step=1)
    eng.apply_gradients()
    assert np.isfinite(eng.read_loss())
    eng.close()


def test_general_kernel_trains_without_deferring(monkeypatch):
    """Under KGE_B200_TRAIN_KERNEL=general no step buckets (kge_train_workspace_bytes is 0), so train_step, the trainer
    at world 1 and the facade run the general kernel and the plain optimizer, as before; the tables agree with the default
    (deferred) steps."""
    from ampligraph_b200.parallel import DataParallelTrainer
    rng = np.random.default_rng(43)
    E, R, B, k, eta = 800, 7, 1500, 24, 5
    t = _dev(_zipf_triples(E, R, B, rng))
    ent, rel = _tables("ComplEx", E, R, k, rng)
    out = {}
    for which in ("default", "general"):
        if which == "general":
            monkeypatch.setenv("KGE_B200_TRAIN_KERNEL", "general")
        eng = _engine("ComplEx", k, eta, E, R, loss="self_adversarial", optimizer="adam")
        assert (int(eng.lib.kge_train_workspace_bytes(eng.h, B)) > 0) == (which == "default")
        eng.set_embeddings(ent, rel)
        for step in range(2):
            launches = eng.launches
            eng.train_step(t, None, seed=2, step=step)
            assert eng.launches - launches == (5 if which == "default" else 2)
        out[which] = [x.cpu().numpy() for x in eng.get_embeddings()] + [eng.read_loss()]
        eng.close()
        dp = DataParallelTrainer(lambda alloc: _engine("ComplEx", k, eta, E, R, loss="self_adversarial", table_alloc=alloc))
        dp.eng.set_embeddings(ent, rel)
        dp.train_step(t, None, seed=2, step=0)
        assert dp.eng._pblock_next is None if which == "general" else dp.eng._pblock_next is not None
        dp.close()
    for got, want, init in zip(out["general"][:2], out["default"][:2], (ent, rel)):
        ok, err = tables_close(got, want, init)
        assert ok, err
    assert abs(out["general"][2] - out["default"][2]) <= 1e-6 * abs(out["default"][2])
