"""Host-side data plumbing either side of the hot path (vectorised numpy/pandas).

* DataIndexer  -- label <-> int32 id mapping with the reference's first-seen order
  (ampligraph/datasets/data_indexer.py:373-428: scan rows, subject then object for
  entities; predicates separately), unknown labels dropped on lookup (:525-542).
* FilterIndex  -- known-true entities per (p,o) / (s,p) (and relations per (s,o)) as CSR, built ONCE, replacing
  the per-batch pandas groupby/reindex + tf.ragged.constant of
  ampligraph/datasets/graph_data_loader.py:287-350, :382-439, :501-521.
"""
import numpy as np
import pandas as pd


def as_triple_array(x, sep="\t"):
    """Accept what the reference's DataSourceIdentifier accepts for an in-memory run
    (ampligraph/datasets/source_identifier.py:25-50, :134-136): a numpy array / nested list, a pandas
    DataFrame, or the path of a csv / txt / gz file with one `sep`-separated triple per line and no header."""
    if isinstance(x, str):
        ext = x.rsplit(".", 1)[-1].lower() if "." in x else ""
        if ext not in ("csv", "txt", "gz"):
            raise ValueError("Unsupported data source file type: %r (expected csv, txt or gz)" % x)
        return pd.read_csv(x, sep=sep, header=None).values
    if isinstance(x, pd.DataFrame):
        return x.values
    return np.asarray(x)


class DataIndexer:
    def __init__(self, X=None):
        self.ent_labels = np.empty(0, dtype=object)
        self.rel_labels = np.empty(0, dtype=object)
        self._ent_index = pd.Index([])
        self._rel_index = pd.Index([])
        if X is not None:
            self.update(X)

    # ids are assigned in first-seen order over s0,o0,s1,o1,... and p0,p1,...
    def update(self, X):
        X = np.asarray(X)
        ents = pd.unique(np.stack([X[:, 0], X[:, 2]], axis=1).ravel())
        rels = pd.unique(X[:, 1])
        new_e = ents[~pd.Index(ents).isin(self._ent_index)] if len(self._ent_index) else ents
        new_r = rels[~pd.Index(rels).isin(self._rel_index)] if len(self._rel_index) else rels
        self.ent_labels = np.concatenate([self.ent_labels, np.asarray(new_e, dtype=object)])
        self.rel_labels = np.concatenate([self.rel_labels, np.asarray(new_r, dtype=object)])
        self._ent_index = pd.Index(self.ent_labels)
        self._rel_index = pd.Index(self.rel_labels)

    def get_entities_count(self):
        return len(self.ent_labels)

    def get_relations_count(self):
        return len(self.rel_labels)

    def get_indexes(self, X, type_of="t", order="raw2ind"):
        """data_indexer.get_indexes: triples / entities / relations, raw->ind or ind->raw."""
        if type_of not in ("t", "e", "r"):
            raise ValueError("type_of must be 't', 'e' or 'r'")
        X = np.asarray(X)
        if order == "raw2ind":
            if type_of == "t":
                s = self._ent_index.get_indexer(X[:, 0])
                p = self._rel_index.get_indexer(X[:, 1])
                o = self._ent_index.get_indexer(X[:, 2])
                ok = (s >= 0) & (p >= 0) & (o >= 0)
                if not ok.all():
                    print("\n%d triples containing invalid keys skipped!\n" % int((~ok).sum()))
                return np.stack([s[ok], p[ok], o[ok]], axis=1).astype(np.int32)
            idx = (self._ent_index if type_of == "e" else self._rel_index).get_indexer(X.ravel())
            return idx[idx >= 0].astype(np.int32)
        if order == "ind2raw":
            if type_of == "t":
                X = X.astype(np.int64)
                return np.stack([self.ent_labels[X[:, 0]], self.rel_labels[X[:, 1]], self.ent_labels[X[:, 2]]], axis=1)
            lab = self.ent_labels if type_of == "e" else self.rel_labels
            return lab[X.astype(np.int64).ravel()]
        raise Exception("No such order available options: ind2raw, raw2ind, instead got {}.".format(order))


class FilterIndex:
    """CSR of known-true subjects per (p,o) and objects per (s,p) over a set of indexed triples; relations per (s,o)
    are grouped on the first 'p' lookup, so callers that rank entities only never pay for them."""

    def __init__(self, indexed_triples, n_ent):
        t = np.unique(np.asarray(indexed_triples, dtype=np.int64).reshape(-1, 3), axis=0)
        self.n_ent = int(n_ent)
        self._sub = self._group(t[:, 1] * self.n_ent + t[:, 2], t[:, 0])  # (p,o) -> subjects
        self._obj = self._group(t[:, 1] * self.n_ent + t[:, 0], t[:, 2])  # (s,p) -> objects
        self._t = t
        self._rel = None  # (s,o) -> relations, built by the first 'p' lookup

    @staticmethod
    def _group(keys, vals):
        order = np.lexsort((vals, keys))
        return keys[order], vals[order].astype(np.int32)

    def lookup(self, triples, side, position_of=None):
        """-> (offsets int64 [b+1], ids int32 [nnz]) for a batch of indexed test triples.
        side: 's' (known subjects), 'o' (known objects) or 'p' (known relations of each (s, o)).
        position_of: optional int array mapping entity id (relation id for 'p') -> candidate position (or -1) when a
        subset of candidates is used (the mapping_dict of AbstractScoringLayer.py:266-275)."""
        t = np.asarray(triples, dtype=np.int64)
        if side == "s":
            keys, vals = self._sub
            q = t[:, 1] * self.n_ent + t[:, 2]
        elif side == "p":
            if self._rel is None:
                self._rel = self._group(self._t[:, 0] * self.n_ent + self._t[:, 2], self._t[:, 1])
            keys, vals = self._rel
            q = t[:, 0] * self.n_ent + t[:, 2]
        else:
            keys, vals = self._obj
            q = t[:, 1] * self.n_ent + t[:, 0]
        lo = np.searchsorted(keys, q, side="left")
        hi = np.searchsorted(keys, q, side="right")
        lens = hi - lo
        off = np.zeros(len(t) + 1, dtype=np.int64)
        np.cumsum(lens, out=off[1:])
        total = int(off[-1])
        # gather the ranges [lo_i, hi_i) without a Python loop
        idx = np.repeat(lo - off[:-1], lens) + np.arange(total, dtype=np.int64)
        ids = vals[idx] if total else np.zeros(0, np.int32)
        if position_of is not None and total:
            pos = position_of[ids]
            keep = pos >= 0
            row = np.repeat(np.arange(len(t)), lens)[keep]
            ids = pos[keep].astype(np.int32)
            off = np.zeros(len(t) + 1, dtype=np.int64)
            np.cumsum(np.bincount(row, minlength=len(t)), out=off[1:])
        return off, np.ascontiguousarray(ids, dtype=np.int32)


NEGATIVE_SAMPLERS = ("uniform", "bernoulli", "pseudo_typed")


def negative_sampler_tables(triples, n_ent, n_rel, sampler="uniform", filtered=False):
    """The host tables of kge_sample_negatives for one fit (DESIGN.md 3.18), from the distinct training triples
    (duplicates count once) -> dict of numpy arrays, None where the sampler does not use them:
      thresholds  uint32 [n_rel] ('bernoulli'): t_p = floor(2^32 |T_p| / (|H_p| + |T_p|)) with H_p (T_p) the distinct
                  subjects (objects) of relation p, so that the subject is replaced with probability tph / (tph + hpt)
                  (Wang et al., AAAI 2014); 2^31 for a relation without triples
      pools       {'s': (offsets int64 [n_rel + 1], ids int32), 'o': ...} ('pseudo_typed'): the sorted distinct subjects
                  (objects) of each relation, the only entities a replaced subject (object) is drawn from
      filter      {'s': (keys int64, values int32), 'o': ...} (filtered): FilterIndex._sub and ._obj of the triples,
                  the lexsorted known (p * n_ent + o, s) and (p * n_ent + s, o) pairs"""
    if sampler not in NEGATIVE_SAMPLERS:
        raise ValueError("negative_sampler must be one of %s, got %r" % (", ".join(map(repr, NEGATIVE_SAMPLERS)), sampler))
    n_ent, n_rel = int(n_ent), int(n_rel)
    t = np.unique(np.asarray(triples, dtype=np.int64).reshape(-1, 3), axis=0)
    pairs = {"s": np.unique(t[:, 1] * n_ent + t[:, 0]), "o": np.unique(t[:, 1] * n_ent + t[:, 2])}  # sorted (p, e)
    count = {side: np.bincount(pairs[side] // n_ent, minlength=n_rel).astype(np.int64) for side in pairs}
    out = {"thresholds": None, "pools": None, "filter": None}
    if sampler == "bernoulli":
        h, o = count["s"], count["o"]
        out["thresholds"] = np.where(h + o > 0, (o << 32) // np.maximum(h + o, 1), 1 << 31).astype(np.uint32)
    if sampler == "pseudo_typed":
        out["pools"] = {}
        for side in ("s", "o"):
            off = np.zeros(n_rel + 1, dtype=np.int64)
            np.cumsum(count[side], out=off[1:])
            out["pools"][side] = (off, (pairs[side] % n_ent).astype(np.int32))
    if filtered:
        f = FilterIndex(t, n_ent)
        out["filter"] = {"s": f._sub, "o": f._obj}
    return out


def query_rows(triples, n_ent, side):
    """The distinct queries of one side of `triples`, (s, p) for side 'o' and (p, o) for side 's', numbered in order of
    first appearance -> (first int64 [n_queries]: the triple where each query first appears, ascending; rows int64
    [len(triples)]: the query number of every triple).  KvsAll's training rows and NSCaching's cache rows."""
    t = np.asarray(triples, dtype=np.int64).reshape(-1, 3)
    keys = t[:, 1] * int(n_ent) + t[:, 0 if side == "o" else 2]
    _, first, inverse = np.unique(keys, return_index=True, return_inverse=True)
    order = np.argsort(first, kind="stable")  # sorted-key number -> first-appearance number
    number = np.empty(len(first), dtype=np.int64)
    number[order] = np.arange(len(first))
    return first[order], number[inverse.reshape(-1)]


def nscaching_tables(triples, n_ent, n_rel, batch_size, filtered=False):
    """The per-fit tables of NSCaching (kge_nscaching_step, DESIGN.md 3.20) for fit's sequential batches of batch_size
    triples -> dict:
      key_rows  int32 [n, 2]: column 0 the subject-replaced cache row of each triple (its (p, o) in order of first
                appearance, query_rows(.., 's')), column 1 the object-replaced one (its (s, p), query_rows(.., 'o'))
      update    uint8 [n, 2]: 1 iff the triple is the first of its batch with that row, the one that refreshes it
      n_keys    (subject-side rows, object-side rows)
      filter    {'s': (keys int64, values int32), 'o': ...} as negative_sampler_tables' (filtered), else None
    n_rel is accepted for symmetry with negative_sampler_tables; the rows only depend on the triples."""
    t = np.asarray(triples, dtype=np.int64).reshape(-1, 3)
    n, batch_size = len(t), int(batch_size)
    key_rows = np.zeros((n, 2), dtype=np.int32)
    update = np.zeros((n, 2), dtype=np.uint8)
    n_keys = []
    batch = np.arange(n, dtype=np.int64) // max(batch_size, 1)
    for col, side in ((0, "s"), (1, "o")):
        first, rows = query_rows(t, n_ent, side)
        key_rows[:, col] = rows
        n_keys.append(len(first))
        _, lead = np.unique(batch * max(len(first), 1) + rows, return_index=True)  # first of each (batch, row)
        update[lead, col] = 1
    out = {"key_rows": key_rows, "update": update, "n_keys": tuple(n_keys), "filter": None}
    if filtered:
        f = FilterIndex(t, n_ent)
        out["filter"] = {"s": f._sub, "o": f._obj}
    return out


def k_vs_all_queries(findex, triples, side):
    """The KvsAll training rows of one side (DESIGN.md 3.13): every distinct (s, p) of `triples` for side 'o', every
    distinct (p, o) for side 's', in order of first appearance, each labelled with its known objects (subjects) in
    `findex` (a FilterIndex of the same triples).  -> (queries int32 [n, 3], offsets int64 [n + 1], ids int32 [nnz]):
    the labels of query i are ids[offsets[i]:offsets[i + 1]], ascending and distinct; the answer column of a query
    holds its first label, so that every column is a valid entity id."""
    t = np.asarray(triples, dtype=np.int64).reshape(-1, 3)
    col = 2 if side == "o" else 0
    first, _ = query_rows(t, findex.n_ent, side)
    queries = np.ascontiguousarray(t[first], dtype=np.int32)
    off, ids = findex.lookup(queries, side)
    queries[:, col] = ids[off[:-1]]
    return queries, off, ids


def reciprocal_triples(triples, n_rel, sides="s", batch_size=None):
    """The side-o rows of reciprocal relations (DESIGN.md 3.17), with n_rel forward relations and row p + n_rel the
    inverse p^-1 of relation p: the forward triple (s, p, o) for side 'o', the inverse (o, p + n_rel, s) for side 's'.
    A subject query of (s, p, o) is the object query of its inverse.  -> int32 [m n, 3], m the number of sides.  With
    both sides, the rows of each batch of batch_size triples (all of them when None) are adjacent, its forward rows
    first, so that batch i of the triples is rows[m i batch_size:m (i + 1) batch_size] with either number of sides."""
    t = np.asarray(triples, dtype=np.int32).reshape(-1, 3)
    inverse = np.ascontiguousarray(t[:, ::-1])
    inverse[:, 1] += np.int32(n_rel)
    if sides == "s":
        return inverse
    if sides == "o":
        return np.ascontiguousarray(t)
    batch = np.arange(len(t)) // (int(batch_size) if batch_size else max(len(t), 1))
    order = np.argsort(np.concatenate([2 * batch, 2 * batch + 1]), kind="stable")
    return np.ascontiguousarray(np.concatenate([t, inverse])[order])


def k_vs_all_steps(n_o, n_s, batch_size):
    """The steps of one KvsAll epoch over n_o side-o and n_s side-s queries -> list of ((o_lo, o_hi), (s_lo, s_hi)).
    A single side (the other count 0) is cut into sequential slices of batch_size queries.  Both sides: S =
    ceil((n_o + n_s) / batch_size) steps, step i taking the queries [floor(i n / S), floor((i + 1) n / S)) of each
    side, so that every step mixes the two in proportion and holds at most batch_size + 1 queries."""
    n_o, n_s, bs = int(n_o), int(n_s), int(batch_size)
    if n_o == 0 or n_s == 0:
        n = n_o + n_s
        cut = [(lo, min(lo + bs, n)) for lo in range(0, n, bs)]
        return [(c, (0, 0)) if n_o else ((0, 0), c) for c in cut]
    S = -(-(n_o + n_s) // bs)
    return [((i * n_o // S, (i + 1) * n_o // S), (i * n_s // S, (i + 1) * n_s // S)) for i in range(S)]
