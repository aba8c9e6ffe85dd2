"""TEST INFRASTRUCTURE: the negative sampler of kge_sample_negatives (DESIGN.md 3.18) restated in plain Python.

Corruption r = j*B + i of positive i = (s, p, o) draws attempt a from Philox4x32-10 (oracle/philox.py) with counter
(r_lo, r_hi | a << 24, step_lo, step_hi) and key (seed_lo, seed_hi).  The side comes from attempt 0: keep = x & 1, or,
with thresholds, the subject is replaced (keep = 0) iff x < thresholds[p].  The entity of attempt a is
pool[(y * len(pool)) >> 32], the pool of (p, replaced side), or (y * n_ent) >> 32 without one.  With a training set,
a corruption that is one of its triples is drawn again from attempt a + 1 while a + 1 < max_attempts; after the last
attempt it is emitted and counted as a miss.  The filter here is a Python set of the training triples, not the sorted
arrays the kernel searches."""
import numpy as np

from oracle import philox

MASK = 0xFFFFFFFF


def sample(triples, eta, n_ent, seed, step, thresholds=None, pools=None, train=None, max_attempts=1):
    """-> (repl int32 [eta*B], keep uint8 [eta*B], misses).  pools: {'s': (offsets, ids), 'o': ...} or None; train:
    the known triples [n, 3] or None (no filter)."""
    t = np.asarray(triples, dtype=np.int64).reshape(-1, 3)
    B = t.shape[0]
    known = None if train is None else set(map(tuple, np.asarray(train, dtype=np.int64).reshape(-1, 3).tolist()))
    repl = np.empty(B * eta, dtype=np.int32)
    keep = np.empty(B * eta, dtype=np.uint8)
    misses = 0
    for r in range(B * eta):
        s, p, o = (int(x) for x in t[r % B])

        def block(a):
            return philox.philox4x32_10((r & MASK, (r >> 32) | (a << 24), step & MASK, step >> 32),
                                        (seed & MASK, seed >> 32))

        x, y, _, _ = block(0)
        k = (1 if x >= int(thresholds[p]) else 0) if thresholds is not None else x & 1
        pool = None
        if pools is not None:
            off, ids = pools["o" if k else "s"]
            if off[p + 1] > off[p]:
                pool = ids[off[p]:off[p + 1]]

        def entity(y):
            return int(pool[(y * len(pool)) >> 32]) if pool is not None else (y * int(n_ent)) >> 32

        c = entity(y)
        a = 0
        while known is not None and ((s, p, c) if k else (c, p, o)) in known:
            if a + 1 >= max_attempts:
                misses += 1
                break
            a += 1
            c = entity(block(a)[1])
        repl[r], keep[r] = c, k
    return repl, keep, misses


def corrupted_triples(triples, eta, repl, keep):
    """[eta*B, 3] corruptions of (repl, keep): keep = 1 replaces the object, 0 the subject."""
    t = np.tile(np.asarray(triples, dtype=np.int64).reshape(-1, 3), (eta, 1))
    out = t.copy()
    k = np.asarray(keep).astype(bool)
    out[k, 2] = repl[k]
    out[~k, 0] = repl[~k]
    return out
