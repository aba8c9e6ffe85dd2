"""TEST INFRASTRUCTURE: NSCaching (kge_nscaching_step, DESIGN.md 3.20) restated in plain Python.

Side 0 replaces the subject and has one cache row per (p, o); side 1 replaces the object and has one per (s, p).  A
step refreshes every row whose update flag is set, then draws the step's corruptions:
  refresh  candidates c = 0, 1, ...: the row's cached ids, then N2 draws (w * n_ent) >> 32, w word j & 3 of Philox4x32-10
           (oracle/philox.py) with counter (row, (j >> 2) | side << 31, step_lo, step_hi) and key (seed_lo,
           seed_hi ^ 0x4E534341).  Duplicates of an earlier candidate, NaN scores and (filter) training triples are
           dropped.  The scores are c_oracle.corruption_scores' (bit-exact fp32); the Gumbel keys score + G are computed
           in float64, G = -log(-log u), u = ((w' >> 9) + 0.5) 2^-23, w' word c & 3 of the block with counter
           (row, (c >> 2) | 1 << 30 | side << 31, step_lo, step_hi).  The N1 largest keys (ties: lower c) are kept, in
           ascending c.
  draw     corruption r = j*B + i: (x, y) of the corruption stream's block, side = x & 1, n = the row's count;
           ids[(y * n) >> 32], or (y * n_ent) >> 32 and a miss when n = 0."""
import math

import numpy as np

from oracle import c_oracle, philox

MASK = 0xFFFFFFFF
KEY_HI = 0x4E534341


def word(seed, step, row, idx, stream, side):
    v = philox.philox4x32_10((row & MASK, (idx >> 2) | (stream << 30) | (side << 31), step & MASK, step >> 32),
                             (seed & MASK, ((seed >> 32) ^ KEY_HI) & MASK))
    return v[idx & 3]


def words(seed, step, row, n, stream, side):
    """word(.., idx, ..) for idx < n, one Philox block per four words."""
    out = []
    for b in range((n + 3) // 4):
        out += philox.philox4x32_10((row & MASK, b | (stream << 30) | (side << 31), step & MASK, step >> 32),
                                    (seed & MASK, ((seed >> 32) ^ KEY_HI) & MASK))
    return out[:n]


def gumbel_of(w):
    """G in float64 from the word w', through the same u as the kernel (u is exact in fp32)."""
    u = ((w >> 9) + 0.5) * 2.0 ** -23
    return -math.log(-math.log(u))


def gumbel(seed, step, row, c, side):
    return gumbel_of(word(seed, step, row, c, 1, side))


def candidates(cached, n2, n_ent, seed, step, row, side):
    return list(int(e) for e in cached) + [(w * int(n_ent)) >> 32 for w in words(seed, step, row, n2, 0, side)]


def refresh_row(model, side, triple, ent, rel, cached, n1, n2, seed, step, row, known=None, max_rel_size=None):
    """One row's refresh -> (kept ids in ascending c, info): info has 'cand' (all candidates), 'valid' (bool),
    'score' (fp32), 'key' (float64, -inf where dropped) and 'kept' (candidate positions).  ent / rel: dense float32
    tables; triple (s, p, o) the positive that refreshes the row; known: a set of training triples, or None."""
    s, p, o = (int(x) for x in triple)
    n_ent = ent.shape[0]
    cand = candidates(cached, n2, n_ent, seed, step, row, side)
    m = len(cand)
    valid = np.ones(m, bool)
    seen = set()
    for c, e in enumerate(cand):
        if e in seen:
            valid[c] = False
        seen.add(e)
        if known is not None and ((e, p, o) if side == 0 else (s, p, e)) in known:
            valid[c] = False
    sc = c_oracle.corruption_scores(model, "s" if side == 0 else "o", ent[s][None], rel[p][None], ent[o][None],
                                    ent[np.asarray(cand, np.int64)], max_rel_size=max_rel_size or rel.shape[0])[0]
    valid &= ~np.isnan(sc)
    key = np.full(m, -np.inf)
    for c, w in enumerate(words(seed, step, row, m, 1, side)):
        if valid[c]:
            key[c] = float(sc[c]) + gumbel_of(w)
    order = sorted((c for c in range(m) if valid[c]), key=lambda c: (-key[c], c))
    kept = sorted(order[:n1])
    return [cand[c] for c in kept], {"cand": cand, "valid": valid, "score": sc, "key": key, "kept": kept}


def refresh(model, triples, key_rows, update, ent, rel, ids, count, n1, n2, seed, step, known=None, max_rel_size=None):
    """Every flagged row's refresh on copies of the caches -> (ids, count, infos): ids[side] [n_keys, n1], count[side]
    [n_keys], infos {(side, row): info}."""
    ids = [np.array(a, copy=True) for a in ids]
    count = [np.array(a, copy=True) for a in count]
    infos = {}
    for i, t in enumerate(np.asarray(triples).reshape(-1, 3)):
        for side in (0, 1):
            if not update[i][side]:
                continue
            row = int(key_rows[i][side])
            kept, info = refresh_row(model, side, t, ent, rel, ids[side][row, :count[side][row]], n1, n2, seed, step, row,
                                     known, max_rel_size)
            ids[side][row, :len(kept)] = kept
            count[side][row] = len(kept)
            infos[(side, row)] = info
    return ids, count, infos


def draw(triples, key_rows, ids, count, eta, n_ent, seed, step):
    """-> (repl int32 [eta*B], keep uint8 [eta*B], misses) from the caches (ids, count)."""
    B = len(triples)
    repl = np.empty(B * eta, np.int32)
    keep = np.empty(B * eta, np.uint8)
    misses = 0
    for r in range(B * eta):
        x, y, _, _ = philox.philox4x32_10((r & MASK, r >> 32, step & MASK, step >> 32), (seed & MASK, seed >> 32))
        side = x & 1
        row = int(key_rows[r % B][side])
        n = int(count[side][row])
        if n > 0:
            repl[r] = ids[side][row][(y * n) >> 32]
        else:
            repl[r] = (y * int(n_ent)) >> 32
            misses += 1
        keep[r] = side
    return repl, keep, misses


def key_error_bound(key):
    """The fp32 error of a kernel key fl(score + G), G = -logf(-logf(u)), against the float64 key of the same u and the
    same (exact) fp32 score.  logf is within 1 ulp (relative 2^-23), so a = logf(u) = log(u)(1 + e1); log(-a) is then
    log(-log u) + log(1 + e1), off by <= 2^-23 (1 + tiny) absolutely, and the second logf adds <= 2^-23 |log(-log u)|;
    the final add rounds once, <= 2^-24 |key|.  With |G| <= 17 this is below 2^-23 (2 + |G|) + 2^-24 |key|; the bound
    returned doubles it for the second-order terms: 2^-22 (2 + |G|) + 2^-23 |key|, with |G| bounded by 17."""
    return 2.0 ** -22 * (2 + 17) + 2.0 ** -23 * abs(key)
