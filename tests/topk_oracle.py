"""Host restatement of the top-k ordering contract (csrc/kge_topk.cu, DESIGN.md 3.6) -- TEST INFRASTRUCTURE.

Score descending; equal scores (float equality: -0 == +0) by position ascending; every NaN equal to every other NaN and
above +inf.  Stated as np.lexsort over (position, order-preserving uint32 image of the score), with no composite key,
so that it checks the kernel's key construction rather than repeating it.
"""
import numpy as np


def order_image(scores):
    """uint32 image of fp32 scores whose unsigned order is the contract's score order (NaN one value, -0 == +0)."""
    s = np.ascontiguousarray(scores, np.float32)
    u = s.view(np.uint32).copy()
    u[np.isnan(s)] = 0x7fc00000
    u[u == 0x80000000] = 0
    return np.where(u & 0x80000000, ~u, u | 0x80000000).astype(np.uint32)


def topk(scores, k, exclude=None):
    """scores [b, n] -> (positions int64 [b, k], values fp32 [b, k]); exclude: None or b iterables of positions to skip
    (positions outside [0, n) are ignored).  Rows with fewer than k eligible positions end in -1 / -inf."""
    s = np.ascontiguousarray(scores, np.float32).reshape(-1, np.shape(scores)[-1])
    b, n = s.shape
    img = order_image(s)
    pos = np.full((b, k), -1, np.int64)
    val = np.full((b, k), -np.inf, np.float32)
    for i in range(b):
        cand = np.arange(n)
        if exclude is not None:
            drop = np.asarray([p for p in exclude[i] if 0 <= p < n], np.int64)
            cand = np.setdiff1d(cand, drop)
        order = cand[np.lexsort((cand, ~img[i, cand]))][:k]
        pos[i, :len(order)] = order
        val[i, :len(order)] = s[i, order]
    return pos, val
