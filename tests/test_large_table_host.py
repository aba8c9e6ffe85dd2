"""large_table_oracle on small tables of the same structure: the expanded oracles equal c_oracle / topk_oracle /
knn_oracle run directly on the full table, and fail once one sentinel's row is swapped for its neighbour's; the
vectorised Philox equals oracle/philox.py; the initialisers' exactness argument holds in exact rational arithmetic."""
from fractions import Fraction

import numpy as np
import pytest
import torch

import knn_oracle
import large_table_oracle as lt
from oracle import c_oracle, philox
from optim_exact_oracle import fma32
from topk_oracle import topk

E, P, BOUNDS = 3000, 37, (1000, 2100)
MODEL, k, R = "ComplEx", 6, 5
K, KP, LD = 2 * k, 8, 16  # the library's ComplEx layout at k = 6: halves of 8 floats


def _setup(seed=0):
    spec = lt.make_spec(K, E=E, P=P, boundaries=BOUNDS, n_random=40, seed=seed)
    table = torch.zeros((E, LD), dtype=torch.float32)
    lt.fill(table, spec, KP, chunk=700)
    t = table.numpy()
    ent = np.concatenate([t[:, :k], t[:, KP:KP + k]], 1)
    rng = np.random.default_rng(seed + 1)
    rel = rng.uniform(-0.5, 0.5, (R, K)).astype(np.float32)
    ids = np.concatenate([spec.sentinels, rng.integers(0, E, 40)])
    b = 24
    trip = np.stack([rng.choice(ids, b), rng.integers(0, R, b), rng.choice(ids, b)], 1).astype(np.int32)
    return spec, table, ent, rel, trip, rng


def test_fill_structure():
    spec, table, ent, _, _, _ = _setup()
    assert len(spec.sentinels) == 3 + 3 + 2 * 7 + 40
    assert np.isin([997, 1003, 2097, 2103, 0, 2, E - 3, E - 1], spec.sentinels).all()
    assert np.isin(spec.sentinels, np.arange(E)).all() and (spec.sentinels[6 + 2 * 7 - 3:-3] > 2103).any()
    assert (ent == spec.rows[spec.src]).all()
    assert len(np.unique(spec.src[np.setdiff1d(np.arange(E), spec.sentinels)])) == P  # every pool row is used
    assert lt.mismatched_rows(table, spec, KP, chunk=512).size == 0
    assert lt.nonzero_rows(table, chunk=512).size == E
    t2 = table.clone()
    t2[1001, 3] = -t2[1001, 3]
    t2[E - 1, KP + 2] += 1.0
    assert lt.mismatched_rows(t2, spec, KP, chunk=512).tolist() == [1001, E - 1]
    # the hash in int64 never wraps: the same map on a large id range as in exact integers
    ids = np.arange(lt.BIG_E - 5, lt.BIG_E, dtype=np.int64)
    want = [((((int(e) * 40503 + 12345) % 2147483647) ^ (((int(e) * 40503 + 12345) % 2147483647) >> 13)) * 48271)
            % 2147483647 for e in ids]
    assert lt.hash_ids(torch.as_tensor(ids)).tolist() == want


@pytest.mark.parametrize("swap", [False, True])
def test_expanded_oracles_equal_direct(swap):
    spec, table, ent, rel, trip, rng = _setup()
    if swap:  # the table the device would hold if one sentinel's row had been written from its neighbour's
        ent = ent.copy()
        ent[1000] = ent[1001]
    same = []
    filters = [sorted(set(rng.choice(np.arange(995, 1006), 4).tolist())) for _ in range(len(trip))]
    for side in ("s", "o"):
        full = c_oracle.corruption_scores(MODEL, side, ent[trip[:, 0]], rel[trip[:, 1]], ent[trip[:, 2]], ent,
                                          max_rel_size=R)
        got = lt.corruption_scores(MODEL, side, spec, rel, trip)
        same.append(got.view(np.uint32).tobytes() == full.view(np.uint32).tobytes())
        win = lt.corruption_scores(MODEL, side, spec, rel, trip, start_id=990, n_cand=30)
        same.append((win.view(np.uint32) == full[:, 990:1020].view(np.uint32)).all())
        for strategy in ("worst", "middle", "best"):
            want = c_oracle.rank_triples(MODEL, side, strategy, ent, rel, trip)
            same.append((lt.ranks(MODEL, side, strategy, spec, rel, trip) == want).all())
        want = c_oracle.rank_triples(MODEL, side, "worst", ent, rel, trip, filters=filters, start_id=990, n_cand=30)
        same.append((lt.ranks(MODEL, side, "worst", spec, rel, trip, filters=filters, start_id=990, n_cand=30)
                     == want).all())
        sub = rng.permutation(np.arange(950, E))[:300].astype(np.int32)
        sub[:2] = (1000, 1001)
        pos = [sorted(set(rng.integers(0, 300, 3).tolist()) | {0}) for _ in range(len(trip))]
        want = c_oracle.rank_triples(MODEL, side, "middle", ent, rel, trip, filters=pos, cand_ids=sub)
        same.append((lt.ranks(MODEL, side, "middle", spec, rel, trip, filters=pos, cand_ids=sub) == want).all())
        wp, wv = topk(full, 50)
        gp, gv = topk(got, 50)
        same.append((wp == gp).all() and (wv.view(np.uint32) == gv.view(np.uint32)).all())
    rows = np.zeros((E, LD), np.float32)
    rows[:, :k], rows[:, KP:KP + k] = ent[:, :k], ent[:, k:]
    q = np.array([999, 1000, 1004, 2100, 5], np.int64)
    for metric in ("euclidean", "manhattan"):
        want = knn_oracle.distances(metric, rows[q], rows)
        got = lt.distances(metric, spec, q, KP, LD)
        same.append((want.view(np.uint32) == got.view(np.uint32)).all())
    if swap:
        # every comparison that sees the swapped row (its column, or a query or window that holds it) fails
        assert not any(same[:2]) and not all(same), same
    else:
        assert all(same), same


def test_ties_are_heavy():
    """Each pool row stands for ~E / P entities: the full-table scores tie in blocks that position order must break."""
    spec, _, _, rel, trip, _ = _setup()
    got = lt.corruption_scores(MODEL, "o", spec, rel, trip[:1])[0]
    _, counts = np.unique(got, return_counts=True)
    assert counts.max() >= E // P // 2


def test_vectorised_philox_matches_paper_statement():
    rng = np.random.default_rng(3)
    ctr = rng.integers(0, 2 ** 32, (50, 4), dtype=np.uint64)
    for seed in (0, 2, 2 ** 40 + 7):
        got = lt.philox4x32_10(ctr[:, 0], ctr[:, 1], ctr[:, 2], ctr[:, 3], seed, seed >> 32)
        for i in range(len(ctr)):
            want = philox.philox4x32_10(ctr[i].tolist(), (seed & philox.MASK, seed >> 32))
            assert tuple(int(g[i]) for g in got) == want


def test_glorot_fma_exact_in_fp64():
    """fmaf(2L, u, -L) with u = m 2^-24 equals fp64's 2L u - L rounded to fp32 once: the fp64 value is exact (checked
    with Fractions) and its single rounding matches a correctly rounded fp32 fma."""
    rng = np.random.default_rng(5)
    limits = [lt.glorot_limit(lt.BIG_E, 2000), lt.glorot_limit(3000, 12), np.float32(0.1), np.float32(1.0)]
    m = np.concatenate([[0, 1, 2 ** 23 - 1, 2 ** 23, 2 ** 23 + 1, 2 ** 24 - 1], rng.integers(0, 2 ** 24, 2000)])
    for L in limits:
        u = (m.astype(np.float64) * 2.0 ** -24).astype(np.float32)
        fp64 = 2.0 * float(L) * u.astype(np.float64) - float(L)
        for mi, v in zip(m[:300], fp64[:300]):
            exact = 2 * Fraction(float(L)) * Fraction(int(mi), 2 ** 24) - Fraction(float(L))
            assert Fraction(float(v)) == exact, (L, mi)
        assert (fp64.astype(np.float32).view(np.uint32) == fma32(2 * L, u, -L).view(np.uint32)).all()
    # uniform [-1/4, 3/4): b - a = 1, the sum (m - 2^22) 2^-24 is exact
    u = (m.astype(np.float64) * 2.0 ** -24).astype(np.float32)
    for mi in m[:300]:
        exact = Fraction(int(mi), 2 ** 24) - Fraction(1, 4)
        assert Fraction(float(np.float32(float(exact)))) == exact
    a = np.float32(-0.25)
    assert ((u.astype(np.float64) + float(a)).astype(np.float32).view(np.uint32)
            == fma32(np.float32(0.75) - a, u, a).view(np.uint32)).all()


def test_initialiser_rows_match_scalar_philox():
    """glorot_row / uniform_row against the scalar generator, element by element, past element 2^31."""
    rows, Kb = lt.BIG_E, 2000
    seed = 6
    for row in (lt.BIG_BOUNDARIES[1], rows - 1):
        g = lt.glorot_row(row, rows, Kb, seed)
        uu = lt.uniform_row(row, Kb, -0.25, 0.75, seed)
        L = float(lt.glorot_limit(rows, Kb))
        for col in (0, 1, 2, 3, 1647, 1648, 1999):
            e = row * Kb + col
            x = philox.philox4x32_10((e >> 2, e >> 34, 0x474C4F52, 0), (seed, 0))
            bits = x[e & 3]
            assert g[col] == np.float32(2 * L * ((bits >> 8) * 2.0 ** -24) - L)
            x = philox.philox4x32_10((e & philox.MASK, e >> 32, 0x494E4954, 0), (seed, 0))
            assert uu[col] == np.float32((x[0] >> 8) * 2.0 ** -24 - 0.25)
