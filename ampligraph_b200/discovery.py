"""Link prediction on a fitted ScoringBasedEmbeddingModel.

* query_topn        -- discovery.query_topn (ampligraph/discovery/discovery.py:985-1168): the top_n completions of
  (head, relation, ?), (?, relation, tail) or (head, ?, tail).  The reference builds every completed triple on the host,
  scores all of them with model.predict and sorts them with np.argsort, one query per call.  Here entity completion is
  one kge_topk call (csrc/kge_topk.cu): the candidates are scored on the device by the exact ranking chain and only the
  top_n leave it.  Relation completion scores the R completed triples with the kernel predict uses and orders them
  with kge_select_topk.
* query_topn_batch  -- extension: many (s, p, ?) or (?, p, o) queries in one call, optionally filtered like evaluate.

Order of the results (both functions): score descending; equal scores by candidate position ascending (the order of
ents_to_consider / rels_to_consider, or of the entity / relation ids); NaN before +inf (DESIGN.md 3.6).
"""
import logging

import numpy as np
import torch

from .datasets import DataIndexer, FilterIndex, as_triple_array

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
    return model.engine.n_ent if kind == "e" else model.engine.n_rel


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
    with model.predict to fp32 rounding; relation-completion scores are model.predict's bit for bit."""
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
        q = _dev(eng, [[h, r, t]], np.int32)
        ids, val = eng.topk(q, side, int(top_n), cand_ids=cand, n_cand=n_cand)
        ids, val = ids[0].cpu().numpy(), val[0].cpu().numpy()
        keep = ids >= 0
        ents = _labels(model, ids[keep], "e")
        rows = [[head, relation, e] for e in ents] if side == "o" else [[e, relation, tail] for e in ents]
    X, S = np.array(rows), val[keep]
    if len(S) == 1:  # :1165
        return X[0], S[0]
    return X, S


def query_topn_batch(model, X, side="o", top_n=10, use_filter=False, ents_to_consider=None):
    """Extension (no reference counterpart): the top_n entities completing each triple of X on `side` -- 'o' answers
    (s, p, ?), 's' answers (?, p, o).  X holds raw triples (labels); the `side` column is ignored (any value).

    use_filter: as in evaluate -- a dict of datasets, or True for X itself; the known-true completions are excluded
    (a (s, p, o) in a dataset removes o from the answers to (s, p, ?) and s from those to (?, p, o)).
    ents_to_consider: candidate entities (default: all).
    Returns (labels [n, top_n] object array, scores [n, top_n] fp32), sorted per row; rows with fewer than top_n
    eligible candidates end in None / -inf.  Every label of the other two columns must be known to the model.

    Under torchrun with data-parallel training the tables are replicated, so every rank answers its calls locally."""
    eng = _check_fitted(model)
    if side not in ("s", "o"):
        raise _error("`side` must be 's' or 'o', got {!r}".format(side))
    if int(top_n) < 1:
        raise _error("`top_n` must be >= 1")
    X = as_triple_array(X)
    if X.ndim != 2 or X.shape[1] < 3:
        raise _error("X must be an array of triples")
    n = len(X)
    keep_col = 0 if side == "o" else 2
    q = np.zeros((n, 3), np.int64)
    q[:, keep_col] = _ids(model, X[:, keep_col], "e")
    q[:, 1] = _ids(model, X[:, 1], "r")
    unseen = (q[:, keep_col] < 0) | (q[:, 1] < 0)
    if unseen.any():
        raise _error("{} queries contain entities or relations not seen by the model".format(int(unseen.sum())))

    cand, n_cand, position_of = None, _count(model, "e"), None
    if ents_to_consider is not None:
        if not isinstance(ents_to_consider, (list, np.ndarray)):
            raise _error("`ents_to_consider` must be a list or numpy array.")
        sub = _ids(model, ents_to_consider, "e")
        if (sub < 0).any():
            raise _error("Entities in `ents_to_consider` have not been seen by the model.")
        cand, n_cand = _dev(eng, sub, np.int32), len(sub)
        position_of = np.full(eng.n_ent, -1, np.int64)
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
        ids, val = eng.topk(_dev(eng, qb, np.int32), side, int(top_n), off, idx, cand_ids=cand, n_cand=n_cand)
        labels[start:start + len(qb)] = _labels(model, ids.cpu().numpy(), "e")
        scores[start:start + len(qb)] = val.cpu().numpy()
    return labels, scores
