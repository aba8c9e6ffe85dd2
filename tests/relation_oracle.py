"""Host restatement of relation prediction, the relation side (side 'p') of kge_rank / kge_corruption_scores /
kge_topk -- TEST INFRASTRUCTURE.

The score of a candidate relation r for the query (s, ?, o) is the canonical triple score of (s, r, o): the C oracle's
kgeo_score_triple (oracle.c_oracle.score_triples) over the completed triples.  The counts are the entity sides' rule
(oracle/kge_oracle.c: kgeo_ranks_side): int32(score * 1000) compared with the positive's, worst / best / middle, and one
'<=' subtraction per filter entry whose candidate position lies in the window.
"""
import numpy as np

from oracle import c_oracle


def candidates(n_rel, cand_ids=None, cand_begin=0, n_cand=None):
    """The candidate relation ids of a call, in position order."""
    if cand_ids is not None:
        return np.asarray(cand_ids, np.int64)
    n_cand = n_rel - cand_begin if n_cand is None else n_cand
    return np.arange(cand_begin, cand_begin + n_cand, dtype=np.int64)


def score_grid(model, ent, rel, triples, cand, max_rel_size=None):
    """fp32 [b, len(cand)]: the canonical score of (s_i, cand[j], o_i)."""
    t = np.asarray(triples, np.int64)
    cand = np.asarray(cand, np.int64)
    b, m = len(t), len(cand)
    full = np.empty((b * m, 3), np.int32)
    full[:, 0] = np.repeat(t[:, 0], m)
    full[:, 1] = np.tile(cand, b)
    full[:, 2] = np.repeat(t[:, 2], m)
    if b * m == 0:
        return np.zeros((b, m), np.float32)
    return c_oracle.score_triples(model, ent, rel, full, max_rel_size).reshape(b, m)


def quantise(x):
    """AbstractScoringLayer.py:11,:201: int32(score * 1000) in fp32, truncated toward zero."""
    return (np.asarray(x, np.float32) * np.float32(1000.0)).astype(np.int32)


def counts(model, ent, rel, triples, filters=None, cand_ids=None, cand_begin=0, n_cand=None, max_rel_size=None):
    """int32 [b, 3]: the raw counters of kge_rank(side 'p'): {#(q_pos < q_c), #(q_pos == q_c), #filtered}.
    filters: None, or per query a list of candidate POSITIONS (relation ids when cand_ids is None); entries outside the
    window are ignored, repeats count once each."""
    t = np.asarray(triples, np.int64)
    cand = candidates(rel.shape[0], cand_ids, cand_begin, n_cand)
    qpos = quantise(c_oracle.score_triples(model, ent, rel, t, max_rel_size))
    qc = quantise(score_grid(model, ent, rel, t, cand, max_rel_size))
    out = np.zeros((len(t), 3), np.int32)
    out[:, 0] = (qpos[:, None] < qc).sum(1)
    out[:, 1] = (qpos[:, None] == qc).sum(1)
    if filters is not None:
        lo = 0 if cand_ids is not None else cand_begin
        for i, f in enumerate(filters):
            for v in f:
                pos = int(v) - lo
                if 0 <= pos < len(cand):
                    out[i, 2] += int(qpos[i] <= qc[i, pos])
    return out


def finalize(cnt, strategy):
    """kge_rank_finalize: ranks (before the caller's +1) from raw counters."""
    gt, eq, fl = cnt[:, 0], cnt[:, 1], cnt[:, 2]
    r = {"best": gt, "middle": gt + (eq + 1) // 2, "worst": gt + eq}[strategy]
    return (r - fl).astype(np.int32)


def ranks(model, strategy, ent, rel, triples, filters=None, cand_ids=None, cand_begin=0, n_cand=None, max_rel_size=None):
    return finalize(counts(model, ent, rel, triples, filters, cand_ids, cand_begin, n_cand, max_rel_size), strategy)
