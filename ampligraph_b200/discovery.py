"""Link prediction on a fitted ScoringBasedEmbeddingModel.

* query_topn        -- discovery.query_topn (ampligraph/discovery/discovery.py:985-1168): the top_n completions of
  (head, relation, ?), (?, relation, tail) or (head, ?, tail).  The reference builds every completed triple on the host,
  scores all of them with model.predict and sorts them with np.argsort, one query per call.  Here entity completion is
  one kge_topk call (csrc/kge_topk.cu): the candidates are scored on the device by the exact ranking chain and only the
  top_n leave it.  Relation completion scores the R completed triples with the kernel predict uses and orders them
  with kge_select_topk.
* query_topn_batch  -- extension: many (s, p, ?), (?, p, o) or (s, ?, o) queries in one call, optionally filtered like
  evaluate.  Relation prediction (s, ?, o) is one kge_topk call on the relation side (csrc/kge_rank_rel.cu).
* find_nearest_neighbours -- discovery.find_nearest_neighbours (discovery.py:1171-1244): the n_neighbors nearest
  entities of each given entity in embedding space, one kge_knn call per batch of queries instead of sklearn
  NearestNeighbors on the host.
* find_duplicates   -- discovery.find_duplicates (discovery.py:714-982): groups of entities, relations or triples whose
  embeddings lie within a tolerance of each other.  tolerance='auto' runs the reference's bisection over the duplicate
  fraction, evaluated on the host from one nearest-other-row kge_knn pass instead of one radius self-join per step.
* find_clusters     -- discovery.find_clusters (discovery.py:546-711): cluster the embeddings of entities, relations or
  triples.  sklearn's DBSCAN (the default) runs on the GPU with sklearn's labels (KGEEngine.dbscan: radius counts,
  then a union-find over the in-radius core pairs, no neighbourhood list stored); any other algorithm runs its
  fit_predict on the host, as in the reference.
* generate_candidates / discover_facts -- discovery.generate_candidates and discover_facts (discovery.py:21-543):
  candidate statements sampled by entity weights, filtered against X, ranked by evaluate.  The networkx statistics of
  the graph strategies come from per-node wedge counts on the GPU (engine.graph_counts, DESIGN.md 3.9); the
  candidates are the reference's, row for row, for a given seed.

Order of the link-prediction results: score descending; equal scores by candidate position ascending (the order of
ents_to_consider / rels_to_consider, or of the entity / relation ids); NaN before +inf (DESIGN.md 3.6).  Distances are
the canonical fp32 chains of kge_knn (DESIGN.md 3.7), equal distances again by candidate position.
"""
import logging

import numpy as np
import torch

from .datasets import DataIndexer, FilterIndex, as_triple_array, reciprocal_triples
from .engine import fp32_floor

logger = logging.getLogger(__name__)

# queries per kge_topk call of query_topn_batch, before the running lists' share of the workspace caps it further
_BATCH_QUERIES = 1024
_LIST_BYTES = 256 << 20


def _error(msg):
    logger.error(msg)
    return ValueError(msg)


def _count(model, kind):
    di = model.data_indexer
    if isinstance(di, DataIndexer):
        return di.get_entities_count() if kind == "e" else di.get_relations_count()
    if kind == "e":
        return model.engine.n_ent
    # with reciprocal relations the second half of the relation table holds the inverses, which are no candidates
    return model.engine.n_rel // 2 if model.reciprocal_relations else model.engine.n_rel


def _ids(model, values, kind):
    """labels -> int64 ids, -1 where the model has not seen the label (ids themselves without an indexer)."""
    di = model.data_indexer
    if isinstance(di, DataIndexer):
        index = di._ent_index if kind == "e" else di._rel_index
        return index.get_indexer(np.asarray(values, dtype=object).ravel()).astype(np.int64)
    v = np.asarray(values).ravel()
    try:
        v = v.astype(np.int64)
    except (TypeError, ValueError):
        return np.full(v.shape, -1, np.int64)
    return np.where((v >= 0) & (v < _count(model, kind)), v, -1)


def _labels(model, ids, kind):
    """ids -> labels (None where id < 0)."""
    ids = np.asarray(ids, np.int64)
    di = model.data_indexer
    lab = (di.ent_labels if kind == "e" else di.rel_labels) if isinstance(di, DataIndexer) else None
    out = np.empty(ids.shape, dtype=object)
    ok = ids >= 0
    out[ok] = lab[ids[ok]] if lab is not None else ids[ok]
    out[~ok] = None
    return out


def _check_fitted(model):
    if not model.is_fitted:
        raise _error("Model is not fitted.")
    eng = model.engine
    if eng.ent_rows != eng.n_ent:
        raise NotImplementedError("link prediction needs the whole entity table on this device; row-sharded tables "
                                  "are not supported")
    return eng


def _dev(eng, a, dtype):
    return torch.as_tensor(np.ascontiguousarray(a, dtype=dtype)).to(eng.device)


def query_topn(model, top_n=10, head=None, relation=None, tail=None, ents_to_consider=None, rels_to_consider=None):
    """discovery.query_topn (discovery.py:985-1168): the top_n completions of the one missing element among head,
    relation and tail, ranked by the model's score.

    Returns (X, S): X [n, 3] the completed triples (labels), S [n] their fp32 scores, n = min(top_n, candidates); as in
    the reference (:1165, np.squeeze) a single result comes back as X [3] and a scalar score.  Known-true triples are
    not filtered out.  Entity-completion scores are those of the ranking kernels (kge_corruption_scores), which agree
    with model.predict to fp32 rounding; relation-completion scores are model.predict's bit for bit.  The batched
    relation prediction, query_topn_batch(side='p'), scores with the canonical triple score of the ranking kernels
    instead: its scores agree with these to about 1e-4 relative, so the two may order near-ties differently."""
    eng = _check_fitted(model)
    if sum(x is None for x in (head, relation, tail)) != 1:  # :1076-1079
        raise _error("Exactly one of `head`, `relation` or `tail` arguments must be None.")
    for value, kind, what in ((head, "e", "Head entity"), (relation, "r", "Relation"), (tail, "e", "Tail entity")):
        if value is not None and _ids(model, [value], kind)[0] < 0:  # :1081-1099
            raise _error("{} `{}` not seen by model".format(what, value))
    for consider, kind, name, what, clash in (
            (ents_to_consider, "e", "ents_to_consider", "Entities", head is not None and tail is not None),
            (rels_to_consider, "r", "rels_to_consider", "Relations", relation is not None)):
        if consider is None:
            continue
        if clash:  # :1103-1106, :1124-1127
            raise _error("Cannot specify `ents_to_consider` and both `subject` and `object` arguments." if kind == "e"
                         else "Cannot specify both `rels_to_consider` and `relation` arguments.")
        if not isinstance(consider, (list, np.ndarray)):
            raise _error("`{}` must be a list or numpy array.".format(name))
        if (_ids(model, consider, kind) < 0).any():
            raise _error("{} in `{}` have not been seen by the model.".format(what, name))
        if len(consider) < top_n:
            logger.warning("`%s` contains less than top_n values, return set will be truncated.", name)

    h = int(_ids(model, [head], "e")[0]) if head is not None else 0
    t = int(_ids(model, [tail], "e")[0]) if tail is not None else 0
    # an empty list means every candidate, as in the reference (:1146, :1150: `rels_to_consider or list(...)`)
    if relation is None:
        rels = _ids(model, rels_to_consider, "r") if rels_to_consider is not None and len(rels_to_consider) else \
            np.arange(_count(model, "r"), dtype=np.int64)
        if len(rels) < top_n and rels_to_consider is None:
            logger.warning("the model knows fewer than top_n relations, return set will be truncated.")
        trip = np.stack([np.full(len(rels), h), rels, np.full(len(rels), t)], 1)
        scores = eng.score(_dev(eng, trip, np.int32))
        pos, val = eng.select_topk(scores.reshape(1, -1).contiguous(), int(top_n))
        pos, val = pos[0].cpu().numpy(), val[0].cpu().numpy()
        keep = pos >= 0
        rows = [[head, r, tail] for r in _labels(model, rels[pos[keep]], "r")]
    else:
        r = int(_ids(model, [relation], "r")[0])
        cand = None
        if ents_to_consider is not None and len(ents_to_consider):
            cand = _dev(eng, _ids(model, ents_to_consider, "e"), np.int32)
            n_cand = cand.numel()
        else:
            n_cand = _count(model, "e")
            if n_cand < top_n:
                logger.warning("the model knows fewer than top_n entities, return set will be truncated.")
        side = "o" if tail is None else "s"
        q, qs = np.array([[h, r, t]], np.int32), side
        if side == "s" and model.reciprocal_relations:  # (?, r, t) is the tail query (t, r^-1, ?)
            q, qs = reciprocal_triples(q, model.max_rel_size, "s"), "o"
        ids, val = eng.topk(_dev(eng, q, np.int32), qs, int(top_n), cand_ids=cand, n_cand=n_cand)
        ids, val = ids[0].cpu().numpy(), val[0].cpu().numpy()
        keep = ids >= 0
        ents = _labels(model, ids[keep], "e")
        rows = [[head, relation, e] for e in ents] if side == "o" else [[e, relation, tail] for e in ents]
    X, S = np.array(rows), val[keep]
    if len(S) == 1:  # :1165
        return X[0], S[0]
    return X, S


def query_topn_batch(model, X, side="o", top_n=10, use_filter=False, ents_to_consider=None, rels_to_consider=None):
    """Extension (no reference counterpart): the top_n completions of each triple of X on `side` -- 'o' answers
    (s, p, ?), 's' answers (?, p, o) (entities), 'p' answers (s, ?, o) (relations).  X holds raw triples (labels); the
    `side` column is ignored (any value).

    use_filter: as in evaluate -- a dict of datasets, or True for X itself; the known-true completions are excluded
    (a (s, p, o) in a dataset removes o from the answers to (s, p, ?), s from those to (?, p, o) and p from those to
    (s, ?, o)).
    ents_to_consider: candidate entities of side 's' / 'o'; rels_to_consider: candidate relations of side 'p' (default:
    all).
    Returns (labels [n, top_n] object array, scores [n, top_n] fp32), sorted per row; rows with fewer than top_n
    eligible candidates end in None / -inf.  Every label of the other two columns must be known to the model.
    Relation scores are the canonical triple scores of the ranking kernels (see query_topn for how they relate to
    model.predict).

    Under torchrun with data-parallel training the tables are replicated, so every rank answers its calls locally."""
    if side not in ("s", "o", "p"):
        raise _error("`side` must be 's', 'o' or 'p', got {!r}".format(side))
    if side == "p" and ents_to_consider is not None:
        raise _error("`ents_to_consider` does not apply to side 'p' (the candidates are relations): use `rels_to_consider`.")
    if side != "p" and rels_to_consider is not None:
        raise _error("`rels_to_consider` applies to side 'p' only (the candidates of side {!r} are entities).".format(side))
    eng = _check_fitted(model)
    if int(top_n) < 1:
        raise _error("`top_n` must be >= 1")
    X = as_triple_array(X)
    if X.ndim != 2 or X.shape[1] < 3:
        raise _error("X must be an array of triples")
    n = len(X)
    q = np.zeros((n, 3), np.int64)
    known = [(0, "e"), (2, "e")] if side == "p" else [(0 if side == "o" else 2, "e"), (1, "r")]
    for col, kind in known:
        q[:, col] = _ids(model, X[:, col], kind)
    unseen = np.zeros(n, bool)
    for col, _ in known:
        unseen |= q[:, col] < 0
    if unseen.any():
        raise _error("{} queries contain entities or relations not seen by the model".format(int(unseen.sum())))

    kind = "r" if side == "p" else "e"
    consider, name, what = (rels_to_consider, "rels_to_consider", "Relations") if side == "p" else \
        (ents_to_consider, "ents_to_consider", "Entities")
    cand, n_cand, position_of = None, _count(model, kind), None
    if consider is not None:
        if not isinstance(consider, (list, np.ndarray)):
            raise _error("`{}` must be a list or numpy array.".format(name))
        sub = _ids(model, consider, kind)
        if (sub < 0).any():
            raise _error("{} in `{}` have not been seen by the model.".format(what, name))
        cand, n_cand = _dev(eng, sub, np.int32), len(sub)
        position_of = np.full(eng.n_rel if side == "p" else eng.n_ent, -1, np.int64)
        position_of[sub] = np.arange(len(sub))
    findex = None
    if isinstance(use_filter, dict) or use_filter is True:
        parts = [X] if use_filter is True else list(use_filter.values())
        findex = FilterIndex(np.concatenate([model._index(p) for p in parts]), eng.n_ent)

    labels = np.empty((n, int(top_n)), dtype=object)
    scores = np.empty((n, int(top_n)), np.float32)
    chunk = max(1, min(_BATCH_QUERIES, _LIST_BYTES // (24 * int(top_n))))
    for start in range(0, n, chunk):
        qb = q[start:start + chunk]
        off = idx = None
        if findex is not None:
            o_np, i_np = findex.lookup(qb, side, position_of)
            off, idx = _dev(eng, o_np, np.int64), _dev(eng, i_np, np.int32)
        qs = side
        if side == "s" and model.reciprocal_relations:  # (?, p, o) is the tail query (o, p^-1, ?), same filter list
            qb, qs = reciprocal_triples(qb, model.max_rel_size, "s"), "o"
        ids, val = eng.topk(_dev(eng, qb, np.int32), qs, int(top_n), off, idx, cand_ids=cand, n_cand=n_cand)
        labels[start:start + len(qb)] = _labels(model, ids.cpu().numpy(), kind)
        scores[start:start + len(qb)] = val.cpu().numpy()
    return labels, scores


# sklearn metric names -> the two chains kge_knn implements ('minkowski' is sklearn's default, p = 2)
_METRICS = {"euclidean": "euclidean", "l2": "euclidean", "minkowski": "euclidean",
            "manhattan": "manhattan", "l1": "manhattan", "cityblock": "manhattan"}


def _metric(metric):
    if isinstance(metric, str) and metric in _METRICS:
        return _METRICS[metric]
    raise NotImplementedError("metric {!r} is not supported: the distances are computed on the GPU, which implements "
                              "{}".format(metric, ", ".join(sorted(_METRICS))))


def _check_finite(points):
    if not bool(torch.isfinite(points).all()):
        raise ValueError("Input contains NaN or infinity: the embeddings are not finite.")


def _query_batches(n, k):
    """[start, stop) ranges of queries per kge_knn call: as query_topn_batch, bounded by the running lists' share."""
    chunk = max(1, min(_BATCH_QUERIES, _LIST_BYTES // (24 * max(int(k), 1))))
    return [(s, min(s + chunk, n)) for s in range(0, n, chunk)]


def find_nearest_neighbours(kge_model, entities, n_neighbors=10, entities_subset=None, metric="euclidean"):
    """discovery.find_nearest_neighbours (discovery.py:1171-1244): the n_neighbors nearest entities of each of
    `entities` in embedding space, among all entities (in id order) or among entities_subset (in its order).

    Returns (neighbors [len(entities), n_neighbors] labels, distances [len(entities), n_neighbors] fp32), each row
    distance ascending, equal distances in candidate order.  As with sklearn's kneighbors(X), an entity is not excluded
    from its own neighbours.  metric: 'euclidean' / 'l2' / 'minkowski' or 'manhattan' / 'l1' / 'cityblock'; anything
    else raises NotImplementedError.  Distances are the canonical fp32 chains (DESIGN.md 3.7)."""
    if not kge_model.is_fitted:  # :1219-1225
        raise AssertionError("KGE model is not fit!")
    if not isinstance(entities, (list, np.ndarray)):
        raise AssertionError("Invalid type for entities! Must be a list or np.array")
    if entities_subset is not None and not isinstance(entities_subset, (list, np.ndarray)):
        raise AssertionError("Invalid type for entities_subset! Must be a list or np.array")
    eng = _check_fitted(kge_model)
    cand, n_cand = None, _count(kge_model, "e")
    if entities_subset is not None:
        sub = _ids(kge_model, entities_subset, "e")
        if (sub < 0).any():
            raise _error("Entities in `entities_subset` have not been seen by the model.")
        cand, n_cand = _dev(eng, sub, np.int32), len(sub)
    if not n_neighbors < n_cand:  # :1233
        raise AssertionError("n_neighbors must be less than the number of entities being fit!")
    if int(n_neighbors) < 1:
        raise ValueError("Expected n_neighbors > 0. Got {}".format(n_neighbors))
    metric = _metric(metric)
    q = _ids(kge_model, entities, "e")
    if (q < 0).any():
        raise _error("Entities in `entities` have not been seen by the model.")
    qd = _dev(eng, q, np.int32)
    _check_finite(eng.ent[qd.long()])
    _check_finite(eng.ent[:n_cand] if cand is None else eng.ent[cand.long()])

    k = int(n_neighbors)
    labels = np.empty((len(q), k), dtype=object)
    dist = np.empty((len(q), k), np.float32)
    for start, stop in _query_batches(len(q), k):
        ids, d = eng.knn(eng.ent, qd[start:stop], k, metric, cand_ids=cand, n_cand=n_cand)
        labels[start:stop] = _labels(kge_model, ids.cpu().numpy(), "e")
        dist[start:stop] = d.cpu().numpy()
    return np.array(labels.tolist()).reshape(len(q), k), dist


def duplicate_fraction(d1, keys):
    """The duplicate fraction of find_duplicates as a function of the tolerance, from the nearest-other-row distances.

    d1[i] = min over rows j != i of d(i, j) (fp32), keys[i] = the label of row i (hashable).  Row i has a radius
    neighbour other than itself iff d1[i] <= tol, and d is symmetric, so the union of the reference's duplicate sets
    (discovery.py:961) is the set of labels of the rows with d1 <= tol: fraction(tol) = that many labels / len(d1).
    Returns fraction(tol), evaluated by a binary search over the per-label minimum of d1."""
    d1 = np.asarray(d1, np.float64)
    group = {}
    g = np.fromiter((group.setdefault(key, len(group)) for key in keys), np.int64, len(d1))
    per_label = np.full(len(group), np.inf)
    np.minimum.at(per_label, g, d1)
    per_label.sort()
    n = len(d1)
    return lambda tol: int(np.searchsorted(per_label, tol, side="right")) / n


def _check_mode(X, mode):
    """The mode and shape checks of find_duplicates / find_clusters (discovery.py:896-908, :686-701) -> X as an array."""
    modes = ("t", "e", "r")
    if mode not in modes:
        raise _error("Argument `mode` must be one of the following: {}.".format(", ".join(modes)))
    X = np.asarray(X)
    if mode == "t" and (len(X.shape) != 2 or X.shape[1] != 3):
        raise _error("For 't' mode the input X must be a matrix with three columns.")
    if mode in ("e", "r") and len(X.shape) != 1:
        raise _error("For 'e' or 'r' mode the input X must be an array.")
    return X


def _row_ids(model, X, mode):
    """[(ids, kind)] of the column blocks of X's embedding rows: (X, mode) for mode 'e' / 'r', the subject, predicate
    and object columns for mode 't'.  Unseen labels raise ValueError."""
    cols = ((X[:, 0], "e"), (X[:, 1], "r"), (X[:, 2], "e")) if mode == "t" else ((X, mode),)
    out = []
    for values, kind in cols:
        ids = _ids(model, values, kind)
        if (ids < 0).any():
            raise _error("{} in X have not been seen by the model.".format("Entities" if kind == "e" else "Relations"))
        out.append((ids, kind))
    return out


def _points(model, eng, X, mode):
    """The embedding rows of X on the device, contiguous fp32: entity / relation table rows (mode 'e' / 'r') or the
    concatenation [s | p | o] of each triple's rows (mode 't').  Unseen labels and non-finite values raise ValueError."""
    blocks = [(eng.ent if kind == "e" else eng.rel)[_dev(eng, ids, np.int64)] for ids, kind in _row_ids(model, X, mode)]
    points = (blocks[0] if len(blocks) == 1 else torch.cat(blocks, 1)).contiguous()
    _check_finite(points)
    return points


def find_duplicates(X, model, mode="e", metric="l2", tolerance="auto", expected_fraction_duplicates=0.1, verbose=False):
    """discovery.find_duplicates (discovery.py:714-982): the groups of rows of X whose embeddings lie within
    `tolerance` of each other -> (set of frozensets of labels (mode 't': of triples as tuples), tolerance).

    mode 'e' / 'r': X is an array of entities / relations; 't': X is [n, 3] triples, embedded as the concatenation of
    the subject, predicate and object rows.  metric as in find_nearest_neighbours.  tolerance='auto' searches it with
    the reference's bisection (scipy.optimize.bisect over [0, largest pairwise euclidean distance], xtol 1e-3, 50
    iterations) for expected_fraction_duplicates; each step is evaluated on the host from one kge_knn pass that finds
    every row's nearest other row (duplicate_fraction).  The duplicates themselves come from one kge_radius_neighbors
    self-join at the final tolerance: d <= tolerance, inclusive, with the same fp32 d as the bisection saw."""
    from scipy import optimize

    if getattr(model, "is_backward", False):
        model = model.model
    if not model.is_fitted:  # :891-894
        raise _error("Model has not been fitted.")
    X = _check_mode(X, mode)
    metric = _metric(metric)
    eng = _check_fitted(model)
    points = _points(model, eng, X, mode)
    n = len(X)
    every = torch.arange(n, dtype=torch.int32, device=eng.device)

    if tolerance == "auto":
        d1 = np.empty(n, np.float32)
        max_distance = 0.0
        for start, stop in _query_batches(n, 1):
            q = every[start:stop]
            # each row's own position is excluded: the nearest OTHER row (a repeated label counts at distance 0)
            off = torch.arange(stop - start + 1, dtype=torch.int64, device=eng.device)
            _, d = eng.knn(points, q, 1, metric, n_cand=n, filt_off=off, filt_idx=q)
            d1[start:stop] = d[:, 0].cpu().numpy()
            # the bracket of :972, spatial.distance_matrix: euclidean whatever the metric
            _, far = eng.knn(points, q, 1, "euclidean", n_cand=n, farthest=True)
            max_distance = max(max_distance, float(far.max()))
        fraction = duplicate_fraction(d1, [tuple(r) for r in X] if mode == "t" else X.tolist())

        def opt(tol, info):  # :953-969
            fraction_duplicates = fraction(tol)
            if verbose:
                info["Nfeval"] += 1
                logger.info("Eval {}: tol: {}, duplicate fraction: {}".format(info["Nfeval"], tol, fraction_duplicates))
            return fraction_duplicates - expected_fraction_duplicates

        tolerance = optimize.bisect(opt, 0.0, max_distance, xtol=1e-3, maxiter=50, args=({"Nfeval": 0},))

    dups = set()
    radius = fp32_floor(tolerance)
    for start, stop in _query_batches(n, 1):
        off, nbr = eng.radius_neighbors(points, every[start:stop], radius, metric, n_cand=n)
        off, nbr = off.cpu().numpy(), nbr.cpu().numpy()
        for i in range(stop - start):
            row = nbr[off[i]:off[i + 1]]
            if len(row) > 1:  # :942-950
                dups.add(frozenset(tuple(X[j]) for j in row) if mode == "t" else frozenset(X[j] for j in row))
    return dups, tolerance


def _dbscan_on_gpu(clustering_algorithm):
    """(eps, min_samples, metric) when find_clusters runs the clustering on the GPU, None when it calls the
    algorithm's own fit_predict on the host.

    On the GPU: None (DBSCAN()'s defaults, without importing sklearn) and objects whose type is exactly
    sklearn.cluster.DBSCAN with metric_params None and a metric of _METRICS; 'minkowski' only with p 2 (euclidean) or
    1 (manhattan) -- sklearn itself rejects p None there, and other p are other metrics.  The other metrics ignore p.
    algorithm, leaf_size and n_jobs do not change sklearn's labels.  A subclass may override fit, so it stays on the
    host with everything else."""
    if clustering_algorithm is None:
        return 0.5, 5, "euclidean"
    try:
        from sklearn.cluster import DBSCAN
    except ImportError:
        return None
    if type(clustering_algorithm) is not DBSCAN or clustering_algorithm.metric_params is not None:
        return None
    metric = clustering_algorithm.metric
    if not isinstance(metric, str) or metric not in _METRICS:
        return None
    if metric == "minkowski":
        p = clustering_algorithm.p
        if p is None or p not in (1, 2):
            return None
        metric = "manhattan" if p == 1 else "euclidean"
    return clustering_algorithm.eps, clustering_algorithm.min_samples, _METRICS[metric]


def _embeddings(model, X, mode):
    """get_embeddings of X as the reference builds them (discovery.py:703-709): dense rows, [s | p | o] for mode 't'."""
    if mode == "t":
        return np.hstack((model.get_embeddings(X[:, 0], embedding_type="e"),
                          model.get_embeddings(X[:, 1], embedding_type="r"),
                          model.get_embeddings(X[:, 2], embedding_type="e")))
    return model.get_embeddings(X, embedding_type=mode)


def find_clusters(X, model, clustering_algorithm=None, mode="e"):
    """discovery.find_clusters (discovery.py:546-711): cluster the embeddings of X -> labels, int64 [len(X)].

    mode 'e' / 'r': X is an array of entities / relations; 't': X is [n, 3] triples, embedded as the concatenation of
    the subject, predicate and object rows.  clustering_algorithm: an object with fit_predict; None means sklearn's
    DBSCAN() (eps 0.5, min_samples 5, euclidean), the reference's default.

    DBSCAN (None, or exactly sklearn.cluster.DBSCAN with a euclidean or manhattan metric) runs on the GPU
    (KGEEngine.dbscan) and returns sklearn's labels for knn's fp32 distances (DESIGN.md 3.8); the estimator then
    carries labels_, core_sample_indices_, components_ (the dense embedding rows of the core samples) and
    n_features_in_, as after its own fit.  Every other algorithm -- KMeans, a cosine DBSCAN, a DBSCAN subclass -- runs
    its fit_predict on the host on the dense embeddings, exactly as the reference does."""
    if getattr(model, "is_backward", False):
        model = model.model
    if not model.is_fitted:  # :676-679
        raise _error("Model has not been fitted.")
    if clustering_algorithm is not None and not hasattr(clustering_algorithm, "fit_predict"):  # :681-684
        raise _error("Clustering algorithm does not have the `fit_predict` method.")
    X = _check_mode(X, mode)
    gpu = _dbscan_on_gpu(clustering_algorithm)
    if gpu is None:
        _row_ids(model, X, mode)  # get_embeddings would drop unseen labels
        return clustering_algorithm.fit_predict(_embeddings(model, X, mode))
    if clustering_algorithm is not None and hasattr(clustering_algorithm, "_validate_params"):
        clustering_algorithm._validate_params()  # sklearn's own errors for eps <= 0, min_samples < 1, ...
    eps, min_samples, metric = gpu
    eng = _check_fitted(model)
    points = _points(model, eng, X, mode)
    labels, core = eng.dbscan(points, eps, min_samples, metric)
    labels = labels.cpu().numpy()
    if clustering_algorithm is not None:  # as DBSCAN.fit leaves them
        core_idx = np.flatnonzero(core.cpu().numpy())
        components = _embeddings(model, X[core_idx], mode)
        clustering_algorithm.labels_ = labels
        clustering_algorithm.core_sample_indices_ = core_idx
        clustering_algorithm.components_ = components if len(core_idx) else np.empty((0, components.shape[1]))
        clustering_algorithm.n_features_in_ = components.shape[1]
    return labels


_CANDIDATE_STRATEGIES = ("random_uniform", "entity_frequency", "graph_degree", "cluster_coefficient",
                         "cluster_triangles", "cluster_squares")


def _first_known(cand, known):
    """The rows _setdiff2d removes (discovery.py:522-543): those whose key is in `known` (sorted, unique) and that are
    the first occurrence of their key within `cand`.  A later repeat of a known row is kept, as in the reference, whose
    cumsum over the [|A|, |B|, 3] comparison marks only the first match of each row of B.  -> bool [len(cand)]."""
    cand = np.asarray(cand, np.int64)
    hit = np.zeros(len(cand), bool)
    if len(known):
        pos = np.minimum(np.searchsorted(known, cand), len(known) - 1)
        hit = known[pos] == cand
    first = np.zeros(len(cand), bool)
    first[np.unique(cand, return_index=True)[1]] = True
    return hit & first


def _setdiff2d(A, B):
    """discovery._setdiff2d (discovery.py:522-543) with sorted int64 row keys instead of the [|A|, |B|, m] comparison
    array: the rows of A, less the first occurrence in A of every row that is also in B."""
    if len(A.shape) != 2 or len(B.shape) != 2:
        raise RuntimeError("Input arrays must be 2-dimensional.")
    rows = np.concatenate([A, B]) if len(A) and len(B) else (A if len(A) else B)
    if len(rows) == 0 or len(A) == 0:
        return A
    codes = np.stack([np.unique(rows[:, c], return_inverse=True)[1].ravel() for c in range(rows.shape[1])], 1)
    key = np.unique(codes, axis=0, return_inverse=True)[1].ravel().astype(np.int64)
    return A[~_first_known(key[:len(A)], np.unique(key[len(A):]))]


def _graph_weights(strategy, s_node, o_node, n_nodes):
    """The per-node statistic C of generate_candidates' graph strategies (discovery.py:457-471), float64 [n_nodes], for
    the undirected graph with one edge {s_node[i], o_node[i]} per triple: nx.Graph.degree (numpy, a self-loop counting
    twice), or nx.clustering / nx.triangles / nx.square_clustering from the GPU counts (engine.graph_counts).  Each
    value is a float64 division of exact integers, so it is networkx's Python int / int bit for bit."""
    if strategy == "graph_degree":
        keys = np.unique(np.minimum(s_node, o_node) * n_nodes + np.maximum(s_node, o_node))
        a, b = keys // n_nodes, keys % n_nodes
        return (np.bincount(a, minlength=n_nodes) + np.bincount(b, minlength=n_nodes)).astype(np.float64)
    from .engine import graph_counts
    triples = np.stack([s_node, np.zeros_like(s_node), o_node], 1)  # the predicate column is not read
    g = {k: v.cpu().numpy() for k, v in graph_counts(triples, n_nodes).items()}
    tri2, d = g["tri2"], g["d"]
    with np.errstate(divide="ignore", invalid="ignore"):
        if strategy == "cluster_triangles":
            return (tri2 // 2).astype(np.float64)
        if strategy == "cluster_coefficient":
            return np.where(tri2 == 0, 0.0, tri2.astype(np.float64) / (d * (d - 1)).astype(np.float64))
        sq, pot = g["sq"], g["pot"]
        return np.where((d > 1) & (pot > 0), sq.astype(np.float64) / pot.astype(np.float64), 0.0)


class _CandidateSource:
    """What generate_candidates derives from X alone, computed once and shared by every relation of discover_facts:
    the entity pools e_s / e_o, their sampling weights and the sorted int64 keys of X's triples.  Nodes are the
    positions in np.unique of X's subject and object columns together."""

    def __init__(self, X, strategy, consolidate_sides):
        X = X[:, :3] if X.shape[1] > 3 else X  # :334-337
        self.X, self.strategy = X, strategy
        self.nodes = np.unique(np.concatenate((X[:, 0], X[:, 2])))
        self.rels = np.unique(X[:, 1])
        s_node, o_node = np.searchsorted(self.nodes, X[:, 0]), np.searchsorted(self.nodes, X[:, 2])
        self.known = np.unique(self._key(s_node, np.searchsorted(self.rels, X[:, 1]), o_node))
        if consolidate_sides:  # :382-387
            self.e_s = self.e_o = self.nodes
        else:
            self.e_s, self.e_o = np.unique(X[:, 0]), np.unique(X[:, 2])
        self.s_node, self.o_node = np.searchsorted(self.nodes, self.e_s), np.searchsorted(self.nodes, self.e_o)
        self.p_s = self.p_o = None
        if strategy == "entity_frequency":  # :433-449
            if consolidate_sides:
                c_s = c_o = np.unique(X[:, [0, 2]], return_counts=True)[1]
            else:
                c_s, c_o = np.unique(X[:, 0], return_counts=True)[1], np.unique(X[:, 2], return_counts=True)[1]
            self.p_s = c_s.astype(np.float64) / np.sum(c_s.astype(np.float64))
            self.p_o = c_o.astype(np.float64) / np.sum(c_o.astype(np.float64))
        elif strategy != "random_uniform":  # :451-477
            C = _graph_weights(strategy, s_node, o_node, len(self.nodes))
            w_s, w_o = C[self.s_node], C[self.o_node]
            self.p_s, self.p_o = w_s / np.sum(w_s), w_o / np.sum(w_o)

    def _key(self, s, r, o):
        n = len(self.nodes)
        return (np.asarray(s, np.int64) * len(self.rels) + np.asarray(r, np.int64)) * n + np.asarray(o, np.int64)

    def generate(self, target_rel, max_candidates, seed):
        """The sampling loop of generate_candidates (:391-431, :479-519) for one target_rel (a label or a list of
        labels, one meshgrid over them), with its own RandomState(seed); the arguments are checked by the caller."""
        if isinstance(max_candidates, float):
            max_candidates = int(max_candidates * len(self.X))
        rel = np.asarray(target_rel).ravel()
        r_pos = np.minimum(np.searchsorted(self.rels, rel), max(len(self.rels) - 1, 0))
        r_id = np.where(self.rels[r_pos] == rel, r_pos, -1) if len(self.rels) else np.full(len(rel), -1)

        rng = np.random.RandomState(seed)
        uniform = self.strategy == "random_uniform"
        sample_size = int(np.sqrt(max_candidates) + 10)
        X_candidates = np.zeros([max_candidates, 3], dtype=object)
        num_retries, max_retries = 0, 5
        start_idx, end_idx = 0, 0
        while end_idx <= max_candidates - 1:
            # choice over positions draws exactly what choice over the labels does: the stream depends on the size
            if uniform:
                i_s = rng.choice(len(self.e_s), size=sample_size, replace=False)
                i_o = rng.choice(len(self.e_o), size=sample_size, replace=False)
            else:
                i_s = rng.choice(len(self.e_s), size=sample_size, replace=True, p=self.p_s)
                i_o = rng.choice(len(self.e_o), size=sample_size, replace=True, p=self.p_o)
            gen = np.array(np.meshgrid(self.e_s[i_s], target_rel, self.e_o[i_o])).T.reshape(-1, 3)
            ids = np.array(np.meshgrid(self.s_node[i_s], r_id, self.o_node[i_o])).T.reshape(-1, 3)
            key = np.where(ids[:, 1] >= 0, self._key(ids[:, 0], ids[:, 1], ids[:, 2]), -1)
            gen = gen[~_first_known(key, self.known)]
            gen = gen[np.where(gen[:, 0] != gen[:, 2])]  # :371-374
            select_idx = min(len(gen), len(X_candidates) - start_idx)
            end_idx = start_idx + select_idx
            X_candidates[start_idx:end_idx, :] = gen[0:select_idx, :]
            start_idx = end_idx
            num_retries += 1
            if num_retries == max_retries:
                break
        return X_candidates[0:end_idx, :]


def _check_candidate_args(rels, target_rel, max_candidates):
    """The checks of generate_candidates after the strategy's (discovery.py:349-363); rels = np.unique(X[:, 1])."""
    if target_rel not in rels:
        logger.warning("Target relation is not found in triples.")  # no error: target_rel may be missing from X
    if not isinstance(max_candidates, (float, int)):
        raise ValueError("Parameter max_candidates must be a float or int.")
    if max_candidates <= 0:
        raise ValueError("Parameter max_candidates must be a positive integer or float in range (0,1].")


def generate_candidates(X, strategy, target_rel, max_candidates, consolidate_sides=False, seed=0):
    """discovery.generate_candidates (discovery.py:274-519): candidate statements (s, target_rel, o) sampled from the
    entities of X by `strategy`, without the triples of X and without reflexive ones -> object array [n, 3],
    n <= max_candidates.

    For a given seed the result is the reference's, row for row.  The sampling is the reference's loop (the same
    np.random.choice calls on a RandomState(seed), which draws the legacy stream np.random.seed(seed) gives, but leaves
    the global RNG alone).  The filter of known triples has _setdiff2d's semantics on sorted int64 keys, without its
    [|A|, |B|, 3] array.  The graph statistics of 'cluster_coefficient', 'cluster_triangles' and 'cluster_squares' are
    computed on the GPU (engine.graph_counts, DESIGN.md 3.9) and equal networkx's bit for bit; 'graph_degree' and
    'entity_frequency' are counted on the host."""
    X = np.asarray(X)
    if strategy not in _CANDIDATE_STRATEGIES:  # :338-347
        raise ValueError("%s is not a valid candidate generation strategy." % strategy)
    _check_candidate_args(np.unique(X[:, 1]), target_rel, max_candidates)  # before the weights, as in the reference
    return _CandidateSource(X, strategy, consolidate_sides).generate(target_rel, max_candidates, seed)


def discover_facts(X, model, top_n=10, strategy="random_uniform", max_candidates=100, target_rel=None, seed=0):
    """discovery.discover_facts (discovery.py:21-271): candidate statements from generate_candidates, ranked by
    model.evaluate against their subject and object corruptions (filtered by X); the candidates whose mean rank is
    <= top_n -> (X_pred object array [n, 3], mean ranks float64 [n]).

    target_rel: a relation label, a list of them (one meshgrid over the list, as in the reference), or None for every
    relation the model knows, in the indexer's order, each sampled with the generator reset to `seed`.  A float
    max_candidates is a fraction of len(X).  The weights and X's keys are computed once per call, and every candidate
    is ranked in one evaluate call (the ranks do not depend on batching).  The 'exhaustive' strategy is rejected, as in
    the reference.

    Deliberate deviations from the reference (DESIGN.md 7):
    * target_rel=None stacks the per-relation results with np.vstack, in relation order; the reference's np.hstack
      raises as soon as two relations discover different numbers of facts.
    * candidates with an entity (or relation) the model has not seen are dropped with a warning before ranking, as the
      reference's docstring promises; its ranks would no longer line up with its candidates.
    * the global numpy RNG is not reseeded."""
    if getattr(model, "is_backward", False):
        model = model.model
    if not model.is_fitted:  # :175-178
        raise _error("Model is not fitted.")
    if strategy not in _CANDIDATE_STRATEGIES:  # :185-195
        raise _error("%s is not a valid strategy." % strategy)
    X = np.asarray(X)
    if isinstance(max_candidates, float):  # :201-207
        max_candidates = int(max_candidates * len(X))
    if isinstance(target_rel, str):
        target_rel = [target_rel]
    known_rels = _labels(model, np.arange(_count(model, "r")), "r").tolist()
    if target_rel is None:  # :212-229
        logger.info("No target relation specified. Using all relations to generate candidate statements.")
        rel_list = known_rels
    else:
        missing_rels = [rel for rel in target_rel if rel not in known_rels]
        if len(missing_rels) > 0:
            raise _error("Target relation(s) not found in model: {}".format(missing_rels))
        rel_list = [target_rel]

    if not isinstance(max_candidates, (float, int)) or max_candidates <= 0:  # before the weights
        _check_candidate_args(np.unique(X[:, 1]), rel_list[0] if rel_list else None, max_candidates)
    source = _CandidateSource(X, strategy, False)
    parts = []
    for relation in rel_list:
        logger.info("Generating candidates for relation: %s" % relation)
        _check_candidate_args(source.rels, relation, max_candidates)
        parts.append(source.generate(relation, max_candidates, seed))
    candidates = np.vstack(parts) if parts else np.empty((0, 3), dtype=object)
    seen = (_ids(model, candidates[:, 0], "e") >= 0) & (_ids(model, candidates[:, 1], "r") >= 0) & \
        (_ids(model, candidates[:, 2], "e") >= 0)
    if not seen.all():
        logger.warning("%d candidate statements contain entities not seen by the model and are dropped.",
                       int((~seen).sum()))
        candidates = candidates[seen]
    if len(candidates) == 0:
        return candidates, np.empty(0, np.float64)
    ranks = model.evaluate(candidates, use_filter={"test": X}, corrupt_side="s,o", verbose=False)
    avg_ranks = np.mean(ranks, axis=1)
    preds = avg_ranks <= top_n
    logger.info("Discovered %d facts" % int(preds.sum()))
    return candidates[preds], avg_ranks[preds]
