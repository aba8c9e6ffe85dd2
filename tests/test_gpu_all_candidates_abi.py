"""The C-ABI refusals and workspace sizes of the three all-candidate training steps (DESIGN.md 3.12 to 3.14):
kge_one_vs_all_step, kge_one_vs_all_relation_step and kge_k_vs_all_step, one table-driven check over the three (a test
per entry point runs it).

Every entry point is checked for the refusals they share, with the return code of each: TransE and RotatE; a bad
reduction; a pending deferred step; a single candidate (n_ent = 1, or n_rel = 1); rows too wide for the tiles (ComplEx
k = 900); B = -1; each null table, gradient and triples pointer; a short and a misaligned workspace; and B = 0 with null
pointers and no workspace, a no-op that leaves g_ent, g_rel and loss_acc untouched.  Cases that trip two refusals pin
their order where the two return different codes.  Then each entry point's own arguments, the engine's own refusals,
and kge_*_workspace_bytes against engine.*_workspace_bytes."""
import ctypes as C

import numpy as np
import pytest
import torch

from ampligraph_b200 import _lib
from ampligraph_b200.engine import (KGEEngine, k_vs_all_workspace_bytes, one_vs_all_relation_workspace_bytes,
                                    one_vs_all_workspace_bytes)

pytestmark = pytest.mark.gpu

INVALID, UNSUPPORTED = _lib.KGE_ERR_INVALID_ARGUMENT, _lib.KGE_ERR_UNSUPPORTED


def _dev(a):
    return torch.as_tensor(a).cuda().contiguous()


def _ptr(x):
    return C.c_void_p(x.data_ptr()) if x is not None else C.c_void_p(0)


def _triples(E, R, B, rng):
    return np.stack([rng.integers(0, E, B), rng.integers(0, R, B), rng.integers(0, E, B)], 1).astype(np.int32)


def _labels(E, R, B, rng):
    """B side-o queries, each with one to three sorted, distinct labels: (queries, offsets, ids) on the device."""
    labels = [sorted(set(rng.integers(0, E, rng.integers(1, 4)).tolist())) for _ in range(B)]
    q = _triples(E, R, B, rng)
    q[:, 2] = [lab[0] for lab in labels]
    off = np.concatenate([[0], np.cumsum([len(lab) for lab in labels])]).astype(np.int64)
    return _dev(q), _dev(off), _dev(np.concatenate(labels).astype(np.int32))


class OneVsAll:
    loss, sizer, formula, n_cand = "multiclass_nll", "kge_one_vs_all_workspace_bytes", one_vs_all_workspace_bytes, "n_ent"
    own = {"sides": 3}
    own_refusals = [{"sides": 0}, {"sides": 4}]
    own_accepted = [{"sides": 1}, {"sides": 2}, {"sides": 3, "reduction": 1}]

    @staticmethod
    def inputs(E, R, B, rng):
        return {"triples": _dev(_triples(E, R, B, rng))}

    @staticmethod
    def call(lib, eng, a):
        return lib.kge_one_vs_all_step(eng.h, a["sides"], a["reduction"], _ptr(a["ent"]), _ptr(a["rel"]),
                                       _ptr(a["g_ent"]), _ptr(a["g_rel"]), _ptr(a["triples"]), a["B"], 0,
                                       _ptr(a["loss"]), _ptr(a["ws"]), a["nbytes"], eng._stream())

    @staticmethod
    def backward(eng, a):
        eng.one_vs_all_backward(a["triples"], "s,o")

    @staticmethod
    def engine_refusals(eng, a):
        with pytest.raises(ValueError, match="one_vs_all"):
            eng.one_vs_all_backward(a["triples"], "p")


class Relation:
    loss, sizer, n_cand = "multiclass_nll", "kge_one_vs_all_relation_workspace_bytes", "n_rel"
    formula = one_vs_all_relation_workspace_bytes
    own = {"weight": 1.0}
    own_refusals = [{"weight": w} for w in (0.0, -1.0, float("nan"), float("inf"))]
    own_accepted = [{"weight": 0.5, "reduction": 1}]
    inputs = OneVsAll.inputs

    @staticmethod
    def call(lib, eng, a):
        return lib.kge_one_vs_all_relation_step(eng.h, a["weight"], a["reduction"], _ptr(a["ent"]), _ptr(a["rel"]),
                                                _ptr(a["g_ent"]), _ptr(a["g_rel"]), _ptr(a["triples"]), a["B"], 0,
                                                _ptr(a["loss"]), _ptr(a["ws"]), a["nbytes"], eng._stream())

    @staticmethod
    def backward(eng, a):
        eng.one_vs_all_relation_backward(a["triples"], 1.0)

    @staticmethod
    def engine_refusals(eng, a):
        pass


class KVsAll:
    loss, sizer, formula, n_cand = "nll", "kge_k_vs_all_workspace_bytes", k_vs_all_workspace_bytes, "n_ent"
    own = {"side": 2, "eps": 0.0}
    own_refusals = [{"side": 0}, {"side": 3}, {"side": 4}, {"eps": -0.1}, {"eps": 1.0}, {"eps": float("nan")},
                    {"off": None}, {"ids": None}]
    own_accepted = [{"side": 1, "reduction": 1, "eps": 0.5}]

    @staticmethod
    def inputs(E, R, B, rng):
        q, off, ids = _labels(E, R, B, rng)
        return {"triples": q, "off": off, "ids": ids}

    @staticmethod
    def call(lib, eng, a):
        return lib.kge_k_vs_all_step(eng.h, a["side"], a["reduction"], a["eps"], _ptr(a["ent"]), _ptr(a["rel"]),
                                     _ptr(a["g_ent"]), _ptr(a["g_rel"]), _ptr(a["triples"]), a["B"], _ptr(a["off"]),
                                     _ptr(a["ids"]), 0, _ptr(a["loss"]), _ptr(a["ws"]), a["nbytes"], eng._stream())

    @staticmethod
    def backward(eng, a):
        eng.k_vs_all_backward(a["triples"], "o", a["off"], a["ids"])

    @staticmethod
    def engine_refusals(eng, a):
        with pytest.raises(ValueError, match="side"):
            eng.k_vs_all_backward(a["triples"], "s,o", a["off"], a["ids"])


ENTRIES = {"kge_one_vs_all_step": OneVsAll, "kge_one_vs_all_relation_step": Relation, "kge_k_vs_all_step": KVsAll}


def _setup(entry, model, k, E, R, B, rng, eta=1):
    """An engine and the arguments of one valid call of B queries, its workspace exactly the size the library asks."""
    lib = _lib.load()
    eng = KGEEngine(model, k, eta, E, R, loss=entry.loss)
    ws = torch.empty(max(int(getattr(lib, entry.sizer)(eng.h, B)), 16), dtype=torch.uint8, device="cuda")
    a = {"ent": eng.ent, "rel": eng.rel, "g_ent": eng.g_ent, "g_rel": eng.g_rel, "loss": eng.loss_acc, "B": B,
         "reduction": 0, "ws": ws, "nbytes": int(getattr(lib, entry.sizer)(eng.h, B)), **entry.own,
         **entry.inputs(E, R, B, rng)}
    return lib, eng, a


def _refused(lib, entry, eng, a, code, fn, **kw):
    rc = entry.call(lib, eng, {**a, **kw})
    assert rc == code, (fn, kw, rc)
    msg = lib.kge_last_error().decode()
    assert fn in msg or "reduction" in msg, (fn, kw, msg)
    return msg


def test_one_vs_all_c_abi_refusals_and_workspace():
    _check_refusals_and_workspace("kge_one_vs_all_step")


def test_relation_c_abi_refusals_and_workspace():
    _check_refusals_and_workspace("kge_one_vs_all_relation_step")


def test_k_vs_all_c_abi_refusals_and_workspace():
    _check_refusals_and_workspace("kge_k_vs_all_step")


def _check_refusals_and_workspace(fn):
    """The one check of every entry point in ENTRIES: the shared refusals, its own, and its workspace size."""
    entry = ENTRIES[fn]
    rng = np.random.default_rng(4)
    # the models without inner-product scores, before any other refusal
    for model in ("TransE", "RotatE"):
        lib, eng, a = _setup(entry, model, 4, 100, 40, 50, rng)
        msg = _refused(lib, entry, eng, a, UNSUPPORTED, fn)
        assert "DistMult, ComplEx and HolE" in msg
        _refused(lib, entry, eng, a, UNSUPPORTED, fn, reduction=2, B=-1, ws=None)
        with pytest.raises(NotImplementedError, match="DistMult, ComplEx and HolE"):
            entry.backward(eng, a)
        eng.close()
    # a single candidate: nothing to rank it against
    E, R = (1, 40) if entry.n_cand == "n_ent" else (100, 1)
    lib, eng, a = _setup(entry, "ComplEx", 8, E, R, 12, rng)
    assert entry.n_cand in _refused(lib, entry, eng, a, INVALID, fn)
    with pytest.raises(ValueError, match=entry.n_cand):
        entry.backward(eng, a)
    eng.close()
    # rows too wide for the kernels' shared-memory tiles; checked after the candidate count, before B and the pointers
    lib, eng, a = _setup(entry, "ComplEx", 900, 100, 40, 50, rng)
    assert "shared-memory" in _refused(lib, entry, eng, a, UNSUPPORTED, fn)
    _refused(lib, entry, eng, a, UNSUPPORTED, fn, B=-1, ent=None, ws=None)
    _refused(lib, entry, eng, a, INVALID, fn, reduction=2)
    with pytest.raises(NotImplementedError, match="shared-memory"):
        entry.backward(eng, a)
    eng.close()
    # the arguments of one call, each refused on its own
    lib, eng, a = _setup(entry, "DistMult", 6, 100, 40, 50, rng)
    for B in (0, 1, 50, 1000, 5000):
        assert getattr(lib, entry.sizer)(eng.h, B) == entry.formula(B, getattr(eng, entry.n_cand), eng.ld), B
    assert getattr(lib, entry.sizer)(eng.h, -1) == 0 and getattr(lib, entry.sizer)(None, 50) == 0
    ws = a["ws"]
    for kw in entry.own_refusals + [
            {"reduction": 2}, {"reduction": -1}, {"B": -1}, {"ent": None}, {"rel": None}, {"g_ent": None},
            {"g_rel": None}, {"triples": None}, {"ws": None}, {"nbytes": a["nbytes"] - 16},
            {"ws": ws[4:], "nbytes": a["nbytes"] - 16},  # not 16-byte aligned
            {"ws": ws[8:], "nbytes": a["nbytes"] - 16}]:
        _refused(lib, entry, eng, a, INVALID, fn, **kw)
    entry.engine_refusals(eng, a)
    # an empty batch is a no-op before the pointers and the workspace are looked at
    before = [x.clone() for x in (eng.g_ent, eng.g_rel, eng.loss_acc)]
    nulls = {key: None for key in ("ent", "rel", "g_ent", "g_rel", "triples", "ws", "off", "ids")}
    assert entry.call(lib, eng, {**a, **nulls, "B": 0, "nbytes": 0}) == _lib.KGE_OK
    launches = eng.launches
    entry.backward(eng, {**a, "triples": a["triples"][:0]} if fn != "kge_k_vs_all_step"
                   else {**a, "triples": a["triples"][:0], "off": a["off"][:1]})
    assert eng.launches == launches  # the engine counts no launch for B = 0 either
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(before, (eng.g_ent, eng.g_rel, eng.loss_acc)))
    for kw in [{}] + entry.own_accepted:
        assert entry.call(lib, eng, {**a, **kw}) == _lib.KGE_OK, kw
    torch.cuda.synchronize()
    assert float(eng.loss_acc[0]) > 0.0
    eng.close()
    # a pending deferred step (the bucketed fused step) is refused, by the engine and by the library
    lib, eng, a = _setup(entry, "ComplEx", 8, 64, 3, 64, rng, eta=4)
    eng.forward_backward(_dev(_triples(64, 3, 64, rng)), None, defer=True)
    if eng._deferred:
        with pytest.raises(ValueError, match="deferred"):
            entry.backward(eng, a)
        eng._deferred = False  # past the engine's own check, into the library's
        with pytest.raises(ValueError, match="deferred"):
            entry.backward(eng, a)
        eng._deferred = True
        assert "deferred" in _refused(lib, entry, eng, a, INVALID, fn)
        assert "deferred" in _refused(lib, entry, eng, a, INVALID, fn, B=-1, ent=None, ws=None)
    eng.apply_gradients()
    eng.close()
