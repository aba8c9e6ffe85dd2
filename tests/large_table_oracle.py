"""large_table_oracle.py -- TEST INFRASTRUCTURE: an entity table past 2^31 elements that the host oracles can still
answer for.

A table of E rows is filled on the device from a few thousand distinct source rows: a pool of P Glorot-scaled rows (P
prime) and one unique row per sentinel id.  Entity e holds pool row h(e) mod P, h a fixed integer hash computed in int64
(no product exceeds 2^47, so the CPU and the GPU agree and no intermediate wraps), unless e is a sentinel: the rows
around the boundaries a test wants to cross, the first and last rows of the table and random ids above the last
boundary.  Every candidate's score (distance) under the canonical chain is then the score of its source row, so the
host oracles run on the P + S source rows only and expand their [b, P + S] results to [b, E] through the id -> source
map (`src`) before the counting, quantising and ordering rules see them.  Nothing copies the table through the host:
`fill` writes it chunk by chunk on the device, and `mismatched_rows` regenerates it chunk by chunk to show which rows
differ from the fill.

The philox4x32_10 here is oracle/philox.py's generator vectorised over numpy uint64 (each 32 x 32-bit product fits):
the initialiser restatements draw one block per element or per four elements of a row.
"""
from types import SimpleNamespace

import numpy as np
import torch

from oracle import c_oracle, philox

# cfg5 at one GPU's share: ComplEx, k = 1000 (row stride 2000 floats), 1.1 M entities.  Row 536,870 holds element 2^30
# (byte 2^32) at column 1,824; row 1,073,741 holds element 2^31 at column 1,648.
BIG_E = 1_100_000
BIG_BOUNDARIES = (536_870, 1_073_741)
BIG_P = 4093


def hash_ids(ids):
    """int64 tensor of ids -> int64 hash in [0, 2^31 - 1); every intermediate stays below 2^47."""
    x = (ids * 40503 + 12345) % 2147483647
    x = x ^ (x >> 13)
    return (x * 48271) % 2147483647


def make_spec(K, E=BIG_E, P=BIG_P, boundaries=BIG_BOUNDARIES, n_random=256, seed=0, lim=None):
    """Source rows and sentinels of a table of E rows of K (dense) columns, entries uniform in (-lim, lim) (default
    Glorot's limit sqrt(6 / (E + K)); the ranking tests want scores that spread over many quantisation bins).
    -> SimpleNamespace(E, K, P, sentinels (sorted int64), rows float32 [P + S, K] (pool rows first), src int64 [E])."""
    rng = np.random.default_rng(seed)
    sent = set(range(3)) | set(range(E - 3, E))
    for b in boundaries:
        sent |= set(range(max(b - 3, 0), min(b + 4, E)))
    top = max(boundaries) + 4
    if top < E:
        sent |= set(rng.choice(np.arange(top, E), min(n_random, E - top), replace=False).tolist())
    sent = np.array(sorted(sent), np.int64)
    lim = np.sqrt(6.0 / (E + K)) if lim is None else lim
    rows = rng.uniform(-lim, lim, (P + len(sent), K)).astype(np.float32)
    assert len(np.unique(rows, axis=0)) == len(rows), "source rows must be distinct"
    src = (hash_ids(torch.arange(E, dtype=torch.int64)) % P).numpy()
    src[sent] = P + np.arange(len(sent))
    return SimpleNamespace(E=E, K=K, P=P, sentinels=sent, rows=rows, src=src)


def padded(rows, kp, ld):
    """Dense [n, halves*k] rows -> the library's padded [n, ld] layout (k columns per half, half stride kp)."""
    n, K = rows.shape
    halves = ld // kp
    k = K // halves
    out = np.zeros((n, ld), np.float32)
    for h in range(halves):
        out[:, h * kp:h * kp + k] = rows[:, h * k:(h + 1) * k]
    return out


def _src_of(ids, spec, sent_dev):
    idx = hash_ids(ids) % spec.P
    pos = torch.searchsorted(sent_dev, ids).clamp_(max=len(sent_dev) - 1)
    hit = sent_dev[pos] == ids
    return torch.where(hit, pos + spec.P, idx)


def _chunks(table, spec, chunk):
    dev = table.device
    sent = torch.as_tensor(spec.sentinels, device=dev)
    for a in range(0, spec.E, chunk):
        ids = torch.arange(a, min(spec.E, a + chunk), dtype=torch.int64, device=dev)
        yield a, ids, _src_of(ids, spec, sent)


def fill(table, spec, kp, chunk=32768):
    """Write every row of `table` ([E, ld] on any device) from its source row, chunk by chunk."""
    assert table.shape[0] == spec.E
    src_rows = torch.as_tensor(padded(spec.rows, kp, table.shape[1]), device=table.device)
    for a, ids, s in _chunks(table, spec, chunk):
        table[a:a + len(ids)] = src_rows[s]


def mismatched_rows(table, spec, kp, chunk=32768):
    """Ids of the rows of `table` that differ (bitwise) from the fill, as a sorted int64 numpy array."""
    src_rows = torch.as_tensor(padded(spec.rows, kp, table.shape[1]), device=table.device)
    bad = []
    for a, ids, s in _chunks(table, spec, chunk):
        got = table[a:a + len(ids)]
        want = src_rows[s]
        if torch.equal(got.view(torch.int32), want.view(torch.int32)):
            continue
        bad.append(ids[(got.view(torch.int32) != want.view(torch.int32)).any(1)].cpu().numpy())
    return np.concatenate(bad) if bad else np.zeros(0, np.int64)


def nonzero_rows(table, chunk=32768):
    """Ids of the rows of a device table with any non-zero element (bits), as a sorted int64 numpy array."""
    out = []
    for a in range(0, table.shape[0], chunk):
        nz = (table[a:a + chunk].view(torch.int32) != 0).any(1).nonzero().flatten()
        if nz.numel():
            out.append((nz + a).cpu().numpy())
    return np.concatenate(out) if out else np.zeros(0, np.int64)


# --------------------------------------------------------------------------
# the expanded oracles
# --------------------------------------------------------------------------
def _query_rows(spec, rel, triples):
    t = np.asarray(triples, np.int64)
    return spec.rows[spec.src[t[:, 0]]], np.asarray(rel, np.float32)[t[:, 1]], spec.rows[spec.src[t[:, 2]]]


def _cand(spec, cand_ids, start_id, n_cand):
    if cand_ids is not None:
        return np.asarray(cand_ids, np.int64)
    n = spec.E - start_id if n_cand is None else n_cand
    return np.arange(start_id, start_id + n, dtype=np.int64)


def source_scores(model, side, spec, rel, triples, max_rel_size=None):
    """c_oracle.corruption_scores of every query against the P + S source rows: fp32 [b, P + S]."""
    es, ep, eo = _query_rows(spec, rel, triples)
    return c_oracle.corruption_scores(model, side, es, ep, eo, spec.rows, max_rel_size=max_rel_size or len(rel))


def corruption_scores(model, side, spec, rel, triples, cand_ids=None, start_id=0, n_cand=None, max_rel_size=None):
    """The [b, n_cand] corruption-score matrix of the candidates: cand_ids, or rows start_id ... start_id + n_cand - 1
    (fp32)."""
    U = source_scores(model, side, spec, rel, triples, max_rel_size)
    return U[:, spec.src[_cand(spec, cand_ids, start_id, n_cand)]]


def ranks(model, side, strategy, spec, rel, triples, filters=None, cand_ids=None, start_id=0, n_cand=None,
          max_rel_size=None):
    """kgeo_ranks_side's rule on the expanded scores: the quantised positive score against every candidate's
    (greater, greater-or-equal, equal), the strategy, then one off per filter entry inside the candidates whose score is
    >= the positive's.  Filter entries are entity ids (a range of rows) or positions into cand_ids (a subset)."""
    mrs = max_rel_size or len(rel)
    es, ep, eo = _query_rows(spec, rel, triples)
    qpos = c_oracle.quantise(c_oracle.score_rows(model, es, ep, eo, mrs))
    qU = c_oracle.quantise(c_oracle.corruption_scores(model, side, es, ep, eo, spec.rows, max_rel_size=mrs))
    cand = _cand(spec, cand_ids, start_id, n_cand)
    src = spec.src[cand]
    out = np.empty(len(es), np.int32)
    for i in range(len(es)):
        qc = qU[i][src]
        gt, ge, eq = int((qpos[i] < qc).sum()), int((qpos[i] <= qc).sum()), int((qpos[i] == qc).sum())
        r = gt if strategy == "best" else gt + (eq + 1) // 2 if strategy == "middle" else ge
        for f in (filters[i] if filters is not None else ()):
            if cand_ids is not None:
                if 0 <= f < len(cand):
                    r -= int(qpos[i] <= qc[f])
            elif start_id <= f < start_id + len(cand):
                r -= int(qpos[i] <= qc[f - start_id])
        out[i] = r
    return out


def distances(metric, spec, query_ids, kp, ld):
    """knn_oracle.distances of the queries' rows against every row of the padded table: fp32 [b, E]."""
    import knn_oracle
    rows = padded(spec.rows, kp, ld)
    D = knn_oracle.distances(metric, rows[spec.src[np.asarray(query_ids, np.int64)]], rows)
    return D[:, spec.src]


# --------------------------------------------------------------------------
# the initialisers' draws (csrc/kge_misc.cu: kge_glorot_kernel, kge_init_table_kernel)
# --------------------------------------------------------------------------
def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """philox.philox4x32_10 on arrays of counter words (uint64 holding 32-bit values); -> four uint64 arrays."""
    m = np.uint64(philox.MASK)
    c = [np.asarray(v, np.uint64) & m for v in (c0, c1, c2, c3)]
    k0, k1 = np.uint64(k0 & philox.MASK), np.uint64(k1 & philox.MASK)
    c0, c1, c2, c3 = np.broadcast_arrays(*c)
    for _ in range(10):
        p0, p1 = np.uint64(philox.M0) * c0, np.uint64(philox.M1) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & m, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & m
        k0, k1 = (k0 + np.uint64(philox.W0)) & m, (k1 + np.uint64(philox.W1)) & m
    return c0, c1, c2, c3


def _elements(row, K):
    return np.uint64(row) * np.uint64(K) + np.arange(K, dtype=np.uint64)


def glorot_limit(rows, K):
    """launch_glorot's limit: sqrt(6 / (rows + K)) in double, rounded to fp32 once."""
    return np.float32(np.sqrt(6.0 / (float(rows) + float(K))))


def glorot_row(row, rows, K, seed):
    """Dense row `row` of kge_glorot_kernel on a [rows, K] table (seed as the library receives it).

    Element e = row K + column takes word e & 3 of the Philox block at counter (e >> 2, e >> 34, 'GLOR', 0), key
    (seed, seed >> 32); u = (bits >> 8) 2^-24 and the value is fmaf(2L, u, -L).  That fma is exact in fp64 followed by
    one rounding to fp32: 2L u = L m 2^-23 with m = bits >> 8 < 2^24 is a product of two 24-bit integers (times a power
    of two), so it is exact in fp64's 53 bits, and the sum 2L u - L = L (m - 2^23) 2^-23 is again L times an integer of
    at most 24 bits, so the fp64 subtraction is exact too.  Rounding that exact value to fp32 is what fmaf does."""
    e = _elements(row, K)
    x = philox4x32_10(e >> np.uint64(2), e >> np.uint64(34), 0x474C4F52, 0, seed, seed >> 32)
    bits = np.choose((e & np.uint64(3)).astype(np.int64), x)
    u = (bits >> np.uint64(8)).astype(np.float64) * 2.0 ** -24
    L = float(glorot_limit(rows, K))
    return (2.0 * L * u - L).astype(np.float32)


def uniform_row(row, K, a, b, seed):
    """Dense row `row` of kge_init_table_kernel's 'uniform' kind: fmaf(b - a, (x >> 8) 2^-24, a), x the first word of
    the Philox block at counter (e, e >> 32, 'INIT', 0).  For a = -1/4, b = 3/4 (b - a = 1) the product is m 2^-24 and
    the sum (m - 2^22) 2^-24 has at most 24 significant bits: exact in fp64 and in fp32 alike, as glorot_row argues."""
    e = _elements(row, K)
    x = philox4x32_10(e, e >> np.uint64(32), 0x494E4954, 0, seed, seed >> 32)[0]
    u = (x >> np.uint64(8)).astype(np.float64) * 2.0 ** -24
    ba = float(np.float32(b) - np.float32(a))
    return (ba * u + float(np.float32(a))).astype(np.float32)
