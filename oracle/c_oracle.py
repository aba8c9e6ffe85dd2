"""ctypes front-end of oracle/kge_oracle.c -- TEST INFRASTRUCTURE.

`build()` compiles the C restatement with gcc (seconds); `lib()` loads it.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "libkge_oracle.so")
MODELS = {"TransE": 0, "DistMult": 1, "ComplEx": 2, "HolE": 3, "RotatE": 4}
SIDES = {"s": 0, "o": 1}
STRATEGIES = {"worst": 0, "best": 1, "middle": 2}
_lib = None


def build(force=False):
    src = os.path.join(_HERE, "kge_oracle.c")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.check_call(["make", "-s", "-C", _HERE] + (["-B"] if force else []))
    return _SO


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(_SO)
        _lib.kgeo_score_triple.restype = C.c_float
        _lib.kgeo_rotate_divisor.restype = C.c_float
        _lib.kgeo_hole_scale.restype = C.c_float
    return _lib


def _f(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t)) if a is not None else None


def sincos(x):
    x = _f(x).ravel()
    s, c = np.empty_like(x), np.empty_like(x)
    fs, fc = C.c_float(), C.c_float()
    L = lib()
    for i, v in enumerate(x):
        L.kgeo_sincosf(C.c_float(float(v)), C.byref(fs), C.byref(fc))
        s[i], c[i] = fs.value, fc.value
    return s, c


def score_rows(model, e_s, e_p, e_o, max_rel_size=1):
    e_s, e_p, e_o = _f(e_s), _f(e_p), _f(e_o)
    n, K = e_s.shape
    L = lib()
    out = np.empty(n, np.float32)
    for i in range(n):
        out[i] = L.kgeo_score_triple(MODELS[model], K, int(max_rel_size), _p(e_s[i], C.c_float),
                                     _p(e_p[i], C.c_float), _p(e_o[i], C.c_float))
    return out


def score_triples(model, ent, rel, triples, max_rel_size=None):
    ent, rel = _f(ent), _f(rel)
    t = np.ascontiguousarray(triples, dtype=np.int32)
    K = ent.shape[1]
    out = np.empty(len(t), np.float32)
    lib().kgeo_score_triples(MODELS[model], K, int(max_rel_size or rel.shape[0]), _p(ent, C.c_float),
                             _p(rel, C.c_float), C.c_int64(K), _p(t, C.c_int32), C.c_int64(len(t)),
                             _p(out, C.c_float))
    return out


def corruption_scores(model, side, e_s, e_p, e_o, cand, max_rel_size=1):
    e_s, e_p, e_o, cand = _f(e_s), _f(e_p), _f(e_o), _f(cand)
    b, K = e_s.shape
    m = cand.shape[0]
    out = np.empty((b, m), np.float32)
    lib().kgeo_corruption_scores(MODELS[model], SIDES[side], K, int(max_rel_size), _p(e_s, C.c_float),
                                 _p(e_p, C.c_float), _p(e_o, C.c_float), C.c_int64(b),
                                 _p(cand, C.c_float), C.c_int64(K), C.c_int64(m), _p(out, C.c_float))
    return out


def quantise(x):
    """kgeo_quantise on every element: int32(fl(x * 1000)) truncated toward zero, saturated, NaN -> 0."""
    x = _f(x)
    out = np.empty(x.shape, np.int32)
    lib().kgeo_quantise_many(_p(x, C.c_float), C.c_int64(x.size), _p(out, C.c_int32))
    return out


def _csr(filters, b):
    if filters is None:
        return None, None
    off = np.zeros(b + 1, np.int64)
    for i, f in enumerate(filters):
        off[i + 1] = off[i] + len(f)
    ids = np.ascontiguousarray(np.concatenate([np.asarray(f, np.int32) for f in filters])
                               if off[-1] else np.zeros(0, np.int32), dtype=np.int32)
    return off, ids


def ranks_side(model, side, strategy, e_s, e_p, e_o, cand, start_id, end_id, filters=None, max_rel_size=1):
    """get_ranks for one side on gathered embeddings; `filters` = list of b id-lists or None."""
    e_s, e_p, e_o, cand = _f(e_s), _f(e_p), _f(e_o), _f(cand)
    b, K = e_s.shape
    off, ids = _csr(filters, b)
    out = np.empty(b, np.int32)
    lib().kgeo_ranks_side(MODELS[model], SIDES[side], STRATEGIES[strategy], K, int(max_rel_size),
                          _p(e_s, C.c_float), _p(e_p, C.c_float), _p(e_o, C.c_float), C.c_int64(b),
                          _p(cand, C.c_float), C.c_int64(K), C.c_int64(cand.shape[0]),
                          C.c_int32(start_id), C.c_int32(end_id), _p(off, C.c_int64), _p(ids, C.c_int32),
                          _p(out, C.c_int32))
    return out


def rank_triples(model, side, strategy, ent, rel, triples, filters=None, cand_ids=None,
                 start_id=0, n_cand=None, max_rel_size=None):
    ent, rel = _f(ent), _f(rel)
    t = np.ascontiguousarray(triples, dtype=np.int32)
    K = ent.shape[1]
    b = len(t)
    off, ids = _csr(filters, b)
    cid = None if cand_ids is None else np.ascontiguousarray(cand_ids, dtype=np.int32)
    if n_cand is None:
        n_cand = len(cid) if cid is not None else ent.shape[0] - start_id
    out = np.empty(b, np.int32)
    lib().kgeo_rank_triples(MODELS[model], SIDES[side], STRATEGIES[strategy], K,
                            int(max_rel_size or rel.shape[0]), _p(ent, C.c_float), _p(rel, C.c_float),
                            C.c_int64(K), _p(t, C.c_int32), C.c_int64(b), _p(cid, C.c_int32),
                            C.c_int64(n_cand), C.c_int32(start_id), _p(off, C.c_int64),
                            _p(ids, C.c_int32), _p(out, C.c_int32))
    return out


def corrupt(pos, eta, keep_subj, repl):
    pos = np.ascontiguousarray(pos, dtype=np.int32)
    ks = np.ascontiguousarray(keep_subj, dtype=np.uint8)
    rp = np.ascontiguousarray(repl, dtype=np.int32)
    out = np.empty((len(pos) * eta, 3), np.int32)
    lib().kgeo_corrupt(_p(pos, C.c_int32), C.c_int64(len(pos)), eta, _p(ks, C.c_uint8),
                       _p(rp, C.c_int32), _p(out, C.c_int32))
    return out
