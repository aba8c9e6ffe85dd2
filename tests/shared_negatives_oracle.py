"""TEST INFRASTRUCTURE: the corruptions of kge_shared_negatives_step (DESIGN.md 3.21) restated in plain Python.

A step's B positives are cut into chunks of C consecutive positives: chunk k = positives [k C, min((k + 1) C, B)).
Chunk k has eta candidates c_{k,j} = (y * n_ent) >> 32, (x, y, ..) the Philox4x32-10 block (oracle/philox.py) of
corruption r = j*B + k*C with counter (r_lo, r_hi, step_lo, step_hi) and key (seed_lo, seed_hi) -- the block
kge_generate_corruptions uses for the chunk's first positive.  Corruption j of positive i replaces the side the
per-positive sampler picks for r = j*B + i: keep = x & 1, or, with thresholds, the subject is replaced (keep = 0) iff
x < thresholds[p].  No filtering: a candidate equal to the positive's own entity or to another candidate is an ordinary
corruption.  The output is the (neg_ent, neg_keep) pair in tile order that exact_oracle.oracle_step and
KGEEngine.forward_backward take."""
import numpy as np

from oracle import philox

MASK = 0xFFFFFFFF


def _block(r, seed, step):
    return philox.philox4x32_10((r & MASK, r >> 32, step & MASK, step >> 32), (seed & MASK, seed >> 32))


def chunk_of(i, chunk):
    """The chunk of positive i."""
    return i // chunk


def candidates(B, chunk, eta, n_ent, seed, step):
    """-> int32 [n_chunks, eta]: c_{k,j}."""
    n_chunks = -(-B // chunk)
    out = np.empty((n_chunks, eta), dtype=np.int32)
    for k in range(n_chunks):
        for j in range(eta):
            out[k, j] = (_block(j * B + k * chunk, seed, step)[1] * int(n_ent)) >> 32
    return out


def sample(triples, eta, n_ent, seed, step, chunk, thresholds=None):
    """-> (neg_ent int32 [eta*B], neg_keep uint8 [eta*B]) in tile order, row j*B + i the j-th corruption of positive i."""
    t = np.asarray(triples, dtype=np.int64).reshape(-1, 3)
    B = t.shape[0]
    cand = candidates(B, chunk, eta, n_ent, seed, step)
    ne = np.empty(B * eta, dtype=np.int32)
    nk = np.empty(B * eta, dtype=np.uint8)
    for j in range(eta):
        for i in range(B):
            r = j * B + i
            x = _block(r, seed, step)[0]
            nk[r] = (1 if x >= int(thresholds[t[i, 1]]) else 0) if thresholds is not None else x & 1
            ne[r] = cand[chunk_of(i, chunk), j]
    return ne, nk
