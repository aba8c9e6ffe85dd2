"""ctypes front-end of tests/knn_oracle.c (the canonical distance chains) -- TEST INFRASTRUCTURE.

`build()` compiles the C file with gcc into tests/_build/ (ignored by git), as oracle/c_oracle.py does for the main
oracle; __graft_entry__.build() calls it.  `lib()` builds it there on first use if that has not happened.  Where the tree
cannot be written, the library is built into a fresh private directory (tempfile.mkdtemp: unique name, mode 0700), never
under a predictable name in a shared directory.
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "knn_oracle.c")
_SO = os.path.join(_HERE, "_build", "libkge_knn_oracle.so")
METRICS = {"euclidean": 0, "manhattan": 1}
_lib = None


def _compile(out):
    tmp = "%s.%d.tmp" % (out, os.getpid())
    subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-shared", "-std=c11", "-ffp-contract=off",
                           "-fno-fast-math", "-Wall", "-o", tmp, _SRC, "-lm"])
    os.replace(tmp, out)
    return out


def build(force=False):
    """Compile tests/_build/libkge_knn_oracle.so if it is missing or older than its source; returns its path."""
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(_SRC):
        os.makedirs(os.path.dirname(_SO), exist_ok=True)
        _compile(_SO)
    return _SO


def lib():
    global _lib
    if _lib is None:
        try:
            so = build()
        except (OSError, subprocess.CalledProcessError):  # read-only tree
            so = _compile(os.path.join(tempfile.mkdtemp(prefix="kge_knn_oracle_"), "libkge_knn_oracle.so"))
        _lib = C.CDLL(so)
        _lib.kgeo_distances.restype = None
        _lib.kgeo_distances.argtypes = [C.c_int, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]
    return _lib


def distances(metric, A, B):
    """[na, nb] fp32 canonical distances between the rows of A [na, K] (queries) and B [nb, K] (candidates)."""
    A = np.ascontiguousarray(A, np.float32)
    B = np.ascontiguousarray(B, np.float32)
    assert A.ndim == 2 and B.ndim == 2 and A.shape[1] == B.shape[1]
    out = np.empty((A.shape[0], B.shape[0]), np.float32)
    lib().kgeo_distances(METRICS[metric], A.shape[1], A.ctypes.data, A.shape[0], B.ctypes.data, B.shape[0], out.ctypes.data)
    return out
