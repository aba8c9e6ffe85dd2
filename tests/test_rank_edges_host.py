"""The quantisation's edges, on the host: the one definition of quantise, and the tables that put chosen scores on its bin
edges, at its saturation and on non-finite values.

A rank is a count of quantise(score) comparisons, quantise(x) = cvt.rzi.s32.f32(fl(x * 1000)): truncated toward zero,
saturated (fl(x * 1000) >= 2^31 is INT32_MAX, <= -2^31 is INT32_MIN) and NaN -> 0.  That is what the GPU's conversion
does; C leaves it undefined outside the int32 range and for NaN, so oracle/kge_oracle.c (kgeo_quantise) states it with
explicit comparisons.  This file restates it in numpy once more and checks the three against each other on a sweep of
the values where a conversion goes wrong.

The score-injecting tables (inject_*) are shared with tests/test_gpu_rank_edges.py: every candidate row carries one
chosen value v in column 0 and the query vector is the unit vector e_0 (TransE / RotatE: the zero vector), so the
candidate's canonical score is a closed form of v (DistMult / ComplEx: v, HolE: fl(scale * v), TransE: -|v|, RotatE:
-sqrt(fl(v^2))),
and each query's positive is one of the candidates, so its quantised score is chosen too.
"""
import numpy as np
import pytest

from oracle import c_oracle

MODELS = ["TransE", "DistMult", "ComplEx", "HolE", "RotatE"]
STRATEGIES = ["worst", "best", "middle"]
INT_MIN, INT_MAX = -2 ** 31, 2 ** 31 - 1
FLT_MAX = np.finfo(np.float32).max
EDGE_N = [0, 1, -1, 2, -2, 999, -999, 2147483, -2147483, 2147484, -2147484]


def quantise(x):
    """int32(fl(x * 1000)): truncated toward zero, saturated to the int32 range, NaN -> 0 (kgeo_quantise)."""
    with np.errstate(over="ignore", invalid="ignore"):
        y = (np.asarray(x, np.float32) * np.float32(1000.0)).astype(np.float64)
    q = np.clip(np.trunc(np.nan_to_num(y, nan=0.0)), INT_MIN, INT_MAX)
    return q.astype(np.int64).astype(np.int32)


def ulps(x, n):
    """the floats within n ulps of float32 x (x included), ascending"""
    x = np.float32(x)
    lo, hi = [x], [x]
    for _ in range(n):
        lo.append(np.nextafter(lo[-1], np.float32(-np.inf)))
        hi.append(np.nextafter(hi[-1], np.float32(np.inf)))
    return np.array(lo[:0:-1] + hi, np.float32)


def edge_values(n_ulps=4):
    """every float within n_ulps of n/1000 for the n of EDGE_N, and -0"""
    v = [ulps(np.float32(n / 1000.0), n_ulps) for n in EDGE_N]
    return np.unique(np.concatenate(v + [np.array([-0.0], np.float32)]))


def saturating_values():
    """the neighbours of +-2147483.648 (where fl(x * 1000) reaches +-2^31), values past it, and +-FLT_MAX"""
    v = [ulps(np.float32(2147483.648), 4), ulps(np.float32(-2147483.648), 4),
         np.array([2147483.5, -2147483.5, 3e6, -3e6, 1e10, -1e10, 1e30, -1e30, FLT_MAX, -FLT_MAX], np.float32)]
    return np.unique(np.concatenate(v))


def nonfinite_values():
    return np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, 1.0005, -1.0005, 2147483.75, -2147483.75], np.float32)


def sweep():
    """+-0, subnormals, the bin-edge neighbours, the saturation neighbours, +-FLT_MAX, +-inf and NaN payloads"""
    tiny = np.array([1, 2, 3, 0x7fffff], np.uint32).view(np.float32)
    nans = np.array([0x7fc00000, 0x7fffffff, 0x7f800001, 0xffc00000, 0xff800001, 0x7fa5a5a5], np.uint32).view(np.float32)
    v = [np.array([0.0, -0.0, np.inf, -np.inf, FLT_MAX, -FLT_MAX], np.float32), tiny, -tiny, nans,
         edge_values(4), saturating_values()]
    return np.concatenate(v).astype(np.float32)


def test_quantise_oracle_numpy_and_closed_form():
    """kgeo_quantise (C, through kgeo_quantise_many) == the numpy restatement on the sweep, and both give the stated
    values at the edges: truncation toward zero, saturation at +-2^31, NaN -> 0."""
    x = sweep()
    got = c_oracle.quantise(x)
    want = quantise(x)
    assert got.dtype == np.int32 and (got == want).all(), x[got != want]
    q = dict(zip(x.view(np.uint32).tolist(), got.tolist()))
    at = lambda v: q[int(np.float32(v).view(np.uint32))]  # noqa: E731
    assert at(np.inf) == INT_MAX and at(FLT_MAX) == INT_MAX and at(-np.inf) == INT_MIN and at(-FLT_MAX) == INT_MIN
    assert all(v == 0 for k, v in q.items() if np.isnan(np.uint32(k).view(np.float32)))
    assert at(-0.0) == 0 and at(np.uint32(1).view(np.float32)) == 0
    # fl(2147483.648 * 1000) is 2^31: the first float that saturates; its lower neighbour truncates to 2147483520
    t = np.float32(2147483.648)
    assert np.float32(t * np.float32(1000)) == np.float32(2 ** 31) and at(t) == INT_MAX and at(-t) == INT_MIN
    assert at(np.nextafter(t, np.float32(0))) == 2147483520
    # bin edges: the float nearest n/1000 and its neighbours truncate to n or toward zero from it
    for n in (1, 2, 999, -1, -999):
        for v in ulps(np.float32(n / 1000.0), 4):
            p = np.float64(np.float32(v * np.float32(1000)))
            assert at(v) == int(np.trunc(p))


# ---------------------------------------------------------------------------------------------------------------------
# score-injecting tables
# ---------------------------------------------------------------------------------------------------------------------
def width(model, k):
    return k if model in ("TransE", "DistMult") else 2 * k


def hole_scale(k):
    return np.float32(c_oracle.lib().kgeo_hole_scale(2 * k))


def closed_score(model, k, v):
    """the canonical score of a candidate row [v, 0, ...] against the injected query vector (the chains start from +0,
    so a -0 entry scores +0 on the bilinear models)"""
    v = np.asarray(v, np.float32)
    if model in ("DistMult", "ComplEx"):
        return v + np.float32(0.0)
    if model == "HolE":
        return (hole_scale(k) * (v + np.float32(0.0))).astype(np.float32)
    if model == "RotatE":  # the modulus sqrt(fl(v^2)): |v| while v^2 neither overflows nor underflows
        with np.errstate(over="ignore"):
            return -np.sqrt(v * v)
    return -np.abs(v)


ANCHOR, POISONED_ANCHOR, FIRST_VALUE_ROW = 0, 1, 2


def inject_tables(model, k, values, E, rng, second=0.0, R=2, poison=False):
    """ent [E, K]: row 0 the anchor (the unit vector e_0, or zeros for TransE / RotatE), row 1 the anchor again (with
    poison: with a NaN in column 1), rows 2.. the values spread over the table in a random order (each at least once) in column 0 and
    `second` in column 1.  rel [R, K]: row 0 the unit vector e_0 (zeros: RotatE's phase 0), row 1 the same with +inf in
    column 1 with poison (RotatE: a copy of row 0 always, a non-finite phase has no defined sine).  Returns (ent, rel, row values)."""
    K = width(model, k)
    unit = model not in ("TransE", "RotatE")
    n = E - FIRST_VALUE_ROW
    vals = np.concatenate([values, rng.choice(values, n - len(values))]).astype(np.float32)
    vals = vals[rng.permutation(n)]
    ent = np.zeros((E, K), np.float32)
    ent[ANCHOR, 0] = 1.0 if unit else 0.0
    ent[POISONED_ANCHOR] = ent[ANCHOR]
    if poison:
        ent[POISONED_ANCHOR, 1] = np.nan
    ent[FIRST_VALUE_ROW:, 0] = vals
    ent[FIRST_VALUE_ROW:, 1] = second
    rel = np.zeros((R, K), np.float32)
    if unit:
        rel[:, 0] = 1.0
        if poison:
            rel[1, 1] = np.inf
    return ent, rel, vals


def inject_triples(E, side, b, rng, poison=True):
    """b queries on `side`: the other entity is the anchor, the positive a value row (the first rows of the table in
    order, then random ones).  With poison, every 7th query uses the poisoned anchor and every 11th the poisoned
    relation: a NaN or inf in the query vector."""
    pos = np.concatenate([np.arange(FIRST_VALUE_ROW, min(E, FIRST_VALUE_ROW + b)),
                          rng.integers(FIRST_VALUE_ROW, E, max(0, b - (E - FIRST_VALUE_ROW)))])[:b]
    other = np.full(b, ANCHOR)
    p = np.zeros(b, np.int64)
    if poison:
        other[::7] = POISONED_ANCHOR
        p[3::11] = 1
    t = np.stack([pos, p, other], 1) if side == "s" else np.stack([other, p, pos], 1)
    return np.ascontiguousarray(t, np.int32)


def closed_counts(model, k, ent, t, side, cand):
    """[b, 3] {greater, equal, 0} from quantise over the closed-form scores (clean queries: anchor, relation 0)"""
    pos = t[:, 0] if side == "s" else t[:, 2]
    qpos = quantise(closed_score(model, k, ent[pos, 0]))
    qc = quantise(closed_score(model, k, ent[cand, 0]))
    out = np.zeros((len(t), 3), np.int32)
    out[:, 0] = (qpos[:, None] < qc[None, :]).sum(1)
    out[:, 1] = (qpos[:, None] == qc[None, :]).sum(1)
    return out


def finalize(cnt, strategy):
    gt, eq, fl = cnt[:, 0], cnt[:, 1], cnt[:, 2]
    return {"best": gt, "middle": gt + (eq + 1) // 2, "worst": gt + eq}[strategy] - fl


@pytest.mark.parametrize("group", ["edges", "saturate"])
@pytest.mark.parametrize("model", MODELS)
def test_injected_scores_closed_form_equals_oracle(model, group):
    """The injection works: the oracle's canonical scores of the injected tables are the closed form bit for bit, and
    the oracle's ranks (kgeo_rank_triples) are the closed form's counts of the restated quantise, on both sides, every
    tie strategy, for the full table and a window."""
    k, E, b = 8, 700, 160
    rng = np.random.default_rng(10 * MODELS.index(model) + ["edges", "saturate"].index(group))
    values = edge_values() if group == "edges" else saturating_values()
    ent, rel, _ = inject_tables(model, k, values, E, rng)
    cand = np.arange(E)
    for side in ("s", "o"):
        t = inject_triples(E, side, b, rng, poison=False)
        pos = t[:, 0] if side == "s" else t[:, 2]
        sc = c_oracle.score_triples(model, ent, rel, t)
        assert (sc.view(np.uint32) == closed_score(model, k, ent[pos, 0]).view(np.uint32)).all()
        cs = c_oracle.corruption_scores(model, side, ent[t[:, 0]], rel[t[:, 1]], ent[t[:, 2]], ent)
        want_cs = np.broadcast_to(closed_score(model, k, ent[:, 0]), cs.shape)
        assert (cs.view(np.uint32) == want_cs.view(np.uint32)).all()
        cnt = closed_counts(model, k, ent, t, side, cand)
        assert (cnt[:, 1] >= 1).all()  # the positive ties with itself
        for strategy in STRATEGIES:
            want = c_oracle.rank_triples(model, side, strategy, ent, rel, t)
            assert (finalize(cnt, strategy) == want).all(), (side, strategy)
        win = closed_counts(model, k, ent, t, side, cand[37:37 + 600])
        assert (finalize(win, "middle") == c_oracle.rank_triples(model, side, "middle", ent, rel, t, start_id=37,
                                                                  n_cand=600)).all()
    # the groups do reach what they are for
    q = quantise(closed_score(model, k, ent[:, 0]))
    if group == "saturate":
        assert (q == INT_MIN).any() and (model in ("TransE", "RotatE") or (q == INT_MAX).any())
    else:
        assert len(np.unique(q)) >= 8


@pytest.mark.parametrize("model", MODELS)
def test_nonfinite_oracle_is_defined(model):
    """Non-finite rows and query vectors: the oracle's ranks are the counts of the restated quantise over its own
    scores, so what the GPU is held to is defined (no conversion of NaN or of an out-of-range value to int)."""
    k, E, b = 8, 600, 140
    rng = np.random.default_rng(7)
    ent, rel, _ = inject_tables(model, k, nonfinite_values(), E, rng, second=0.25, poison=True)
    for side in ("s", "o"):
        t = inject_triples(E, side, b, rng)
        qpos = quantise(c_oracle.score_triples(model, ent, rel, t))
        qc = quantise(c_oracle.corruption_scores(model, side, ent[t[:, 0]], rel[t[:, 1]], ent[t[:, 2]], ent))
        cnt = np.stack([(qpos[:, None] < qc).sum(1), (qpos[:, None] == qc).sum(1), np.zeros(b, np.int64)], 1)
        for strategy in STRATEGIES:
            assert (finalize(cnt, strategy) == c_oracle.rank_triples(model, side, strategy, ent, rel, t)).all()
        with np.errstate(invalid="ignore"):
            assert np.isnan(c_oracle.score_triples(model, ent, rel, t[::7])).all()  # the poisoned anchor poisons the query
