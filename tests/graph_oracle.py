"""Host restatement of kge_graph_counts (DESIGN.md 3.9) from row blocks of P = A A, with scipy.

A is the 0/1 adjacency of the undirected simple graph of the edges {s[i], o[i]}: repeated edges and both directions
count once, self-loops are removed.  For a node v, row v of P holds P(v, y) = |N(v) & N(y)| (P(v, v) = d(v)), so
  tri2[v] = sum_y P(v, y) A(v, y)
  sq[v]   = sum_{y != v} P(v, y) (P(v, y) - 1) / 2 = sum_y P(v, y) (P(v, y) - 1) / 2 - d(v) (d(v) - 1) / 2
  pot[v]  = (A d)[v] (d(v) - 1) - d(v) (d(v) - 1) - tri2[v] - sq[v]
Rows are taken in blocks of bounded wedge count, so P never exists whole."""
import numpy as np
import scipy.sparse as sp


def adjacency(s, o, n):
    """(A as int64 CSR without self-loops, networkx degree with a self-loop counting twice)."""
    s, o = np.asarray(s, np.int64), np.asarray(o, np.int64)
    keys = np.unique(np.minimum(s, o) * n + np.maximum(s, o))
    a, b = keys // n, keys % n
    degree = np.bincount(a, minlength=n) + np.bincount(b, minlength=n)
    a, b = a[a != b], b[a != b]
    A = sp.csr_matrix((np.ones(2 * len(a), np.int64), (np.concatenate([a, b]), np.concatenate([b, a]))), shape=(n, n))
    return A, degree


def counts(s, o, n, wedges_per_block=1 << 24):
    """-> dict of int64 [n]: degree, d, tri2, sq, pot."""
    A, degree = adjacency(s, o, n)
    d = np.diff(A.indptr).astype(np.int64)
    nd = A @ d  # sum of the neighbours' degrees = wedges through each node
    tri2, sq = np.zeros(n, np.int64), np.zeros(n, np.int64)
    start = 0
    while start < n:
        stop = start + 1
        budget = nd[start]
        while stop < n and budget + nd[stop] <= wedges_per_block:
            budget += nd[stop]
            stop += 1
        P = (A[start:stop] @ A).tocsr()
        tri2[start:stop] = np.asarray(P.multiply(A[start:stop]).sum(1)).ravel()
        P.data = P.data * (P.data - 1) // 2
        sq[start:stop] = np.asarray(P.sum(1)).ravel()
        start = stop
    sq -= d * (d - 1) // 2
    pot = nd * (d - 1) - d * (d - 1) - tri2 - sq
    return {"degree": degree, "d": d, "tri2": tri2, "sq": sq, "pot": pot}


def networkx_stats(c):
    """nx.triangles, nx.clustering and nx.square_clustering (networkx 3.x) as float64 [n] from counts()."""
    tri2, d, sq, pot = c["tri2"], c["d"], c["sq"], c["pot"]
    with np.errstate(divide="ignore", invalid="ignore"):
        clustering = np.where(tri2 == 0, 0.0, tri2.astype(np.float64) / (d * (d - 1)).astype(np.float64))
        square = np.where((d > 1) & (pot > 0), sq.astype(np.float64) / pot.astype(np.float64), 0.0)
    return tri2 // 2, clustering, square


def complete_bipartite_2(m):
    """Closed-form counts of K_{2,m} (nodes 0 and 1 the hubs, 2 .. m+1 the leaves): for the hubs tri2 = 0,
    sq = pot = m (m - 1) / 2 (the other hub shares all m leaves); for a leaf tri2 = 0, sq = pot = m - 1 (every other
    leaf shares both hubs).  -> (edges s, o, counts)."""
    leaves = np.arange(2, m + 2, dtype=np.int64)
    s, o = np.concatenate([np.zeros(m, np.int64), np.ones(m, np.int64)]), np.concatenate([leaves, leaves])
    n = m + 2
    d = np.full(n, 2, np.int64)
    d[:2] = m
    tri2 = np.zeros(n, np.int64)
    sq = np.full(n, m - 1, np.int64)
    sq[:2] = m * (m - 1) // 2
    return s, o, {"degree": d.copy(), "d": d, "tri2": tri2, "sq": sq, "pot": sq.copy()}
