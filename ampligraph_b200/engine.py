"""KGEEngine: device-memory owner + thin call layer over the C-ABI.

PyTorch tensors hold every byte of device memory (tables, gradient accumulators,
optimizer slots, batches, outputs); all arithmetic happens in libkge_b200.so.
This is the object the reference-facing facade
(ampligraph_b200.latent_features.ScoringBasedEmbeddingModel) drives from its
fit / predict / evaluate loops, mirroring train_function / predict_function /
test_function of the reference (models/ScoringBasedEmbeddingModel.py:443, :1719, :1387).
"""
import ctypes as C
import os

import numpy as np
import torch

from . import _lib


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _metric(metric):
    if metric not in _lib.METRICS:
        raise ValueError("unknown metric %r; supported: %s" % (metric, ", ".join(_lib.METRICS)))
    return _lib.METRICS[metric]


def fp32_floor(x):
    """The largest fp32 value not above the Python number x: for every fp32 d, d <= fp32_floor(x) iff d <= x."""
    with np.errstate(over="ignore"):  # beyond the fp32 range: +inf, stepped down to the largest finite value
        r = np.float32(x)
    if float(r) > float(x):
        r = np.nextafter(r, np.float32(-np.inf))
    return float(r)


def optimizer_slots(cfg):
    """The slot buffers an optimizer config uses (kge_b200.h, kge_optimizer_config; the library's uses_slot0 / uses_slot1)
    -> (initial value of slot 0, of slot 1), None for a slot the kind does not use."""
    O = _lib.OPTIMIZERS
    s0 = None if cfg.kind == O["sgd"] and cfg.momentum == 0.0 else 0.0
    if cfg.kind == O["adagrad"]:
        s0 = float(cfg.initial_accumulator_value)
    s1 = 0.0 if (cfg.kind in (O["adam"], O["adadelta"], O["adamax"])
                 or (cfg.kind == O["rmsprop"] and (cfg.centered or cfg.momentum != 0.0))) else None
    return s0, s1


RHO_DEFAULT = {"rmsprop": 0.9, "adadelta": 0.95}  # Keras legacy defaults; unused by the other kinds


def one_vs_all_splits(B, n_ent):
    """Entity ranges per 32-query tile of the 1vsAll stats and dQ passes (kge_train_1vsall.cu, one_vs_all_splits):
    enough for about 264 CTAs, at most 64 and at most one per 32-entity tile."""
    n_qt, n_et = -(-int(B) // 32), -(-int(n_ent) // 32)
    s = -(-264 // n_qt) if n_qt > 0 else 1
    return max(1, min(s, 64, n_et))


def one_vs_all_workspace_bytes(B, n_ent, ld):
    """kge_one_vs_all_workspace_bytes(h, B) for a handle of n_ent entities and rows of ld floats: both sides' query
    vectors [B, ld], the quantised positive scores [B], the per-split maxima and sums [nsplit, B], three [B] row arrays
    and the per-split partial query gradients [nsplit, B, ld], each region padded to 16 bytes."""
    r16 = lambda n: (n + 15) // 16 * 16
    B, ns = int(B), one_vs_all_splits(B, n_ent)
    rows, col = 4 * B * int(ld), 4 * B
    return 2 * r16(rows) + r16(col) + 2 * r16(ns * col) + 3 * r16(col) + r16(ns * rows)


def one_vs_all_relation_workspace_bytes(B, n_rel, ld):
    """kge_one_vs_all_relation_workspace_bytes(h, B) for a handle of n_rel relations and rows of ld floats: the relation
    queries [B, ld], the per-split maxima and sums [nsplit, B], three [B] row arrays, the per-split partial query
    gradients [nsplit, B, ld] and, when the dX pass splits the query tiles (xsplit > 1), its partial relation rows
    [xsplit, n_rel, ld], each region padded to 16 bytes."""
    r16 = lambda n: (n + 15) // 16 * 16
    B, ns, xs = int(B), one_vs_all_splits(B, n_rel), one_vs_all_splits(n_rel, B)
    rows, col = 4 * B * int(ld), 4 * B
    return (r16(rows) + 2 * r16(ns * col) + 3 * r16(col) + r16(ns * rows)
            + (r16(4 * xs * int(n_rel) * int(ld)) if xs > 1 else 0))


def k_vs_all_workspace_bytes(B, n_ent, ld):
    """kge_k_vs_all_workspace_bytes(h, B): both sides' query vectors [B, ld], the quantised positive scores [B] and the
    per-split partial query gradients [nsplit, B, ld], each region padded to 16 bytes (no row statistics)."""
    r16 = lambda n: (n + 15) // 16 * 16
    B, ns = int(B), one_vs_all_splits(B, n_ent)
    rows = 4 * B * int(ld)
    return 2 * r16(rows) + r16(4 * B) + r16(ns * rows)


INT32_MAX = 2 ** 31 - 1
DBSCAN_BATCH = 1024  # queries per kge_radius_* call of KGEEngine.dbscan (discovery.find_duplicates' batch)


def dbscan_labels(core, root, border_root):
    """sklearn DBSCAN's labels from the union-find result, on any device (O(n) plumbing of KGEEngine.dbscan).

    core: bool [n].  root: int [n], for every core row the smallest index of its component (the component's seed);
    other entries are not read.  border_root: int [n], for every non-core row the smallest root among its core
    neighbours, or a value outside [0, n) if it has none; core entries are not read.
    Clusters are numbered 0, 1, ... in ascending seed order (an exclusive cumsum over the roots, the core rows with
    root[x] == x).  A core row takes its component's number, a non-core row that of border_root, or -1 (noise).
    -> int64 [n]."""
    n = core.numel()
    idx = torch.arange(n, device=core.device)
    root, border_root = root.long(), border_root.long()
    is_root = (core & (root == idx)).long()
    number = torch.cumsum(is_root, 0) - is_root
    labels = torch.full((n,), -1, dtype=torch.int64, device=core.device)
    labels[core] = number[root[core]]
    border = ~core & (border_root >= 0) & (border_root < n)
    labels[border] = number[border_root[border]]
    return labels


def graph_csr(triples, n_nodes, device=None):
    """The CSR of graph_counts, built on the device with torch: (degree, d, offsets int64 [n + 1], nbr int32, order
    int32 [n]) for the undirected simple graph of the edges {s, o} of indexed triples [n, 3] (a CUDA tensor or a host
    array).  degree is nx.Graph.degree (a self-loop counts twice); d = |N(v)| leaves self-loops out; nbr lists both
    directions of each unique non-loop edge, sorted; order is the heaviest-first processing order (descending sum of
    the neighbours' d, the wedges through v).  device: default that of a CUDA `triples`, else the current one."""
    if device is not None:
        dev = torch.device(device)
    elif torch.is_tensor(triples) and triples.is_cuda:
        dev = triples.device
    else:
        dev = torch.device("cuda", torch.cuda.current_device())
    n = int(n_nodes)
    if not 0 <= n < 2 ** 31:
        raise ValueError("graph_counts: n_nodes must be in [0, 2^31), got %d" % n)
    t = (triples if torch.is_tensor(triples) else torch.as_tensor(np.ascontiguousarray(triples))).to(dev)
    if t.dim() != 2 or t.shape[1] != 3:
        raise ValueError("graph_counts: triples must be [n, 3]")
    s, o = t[:, 0].long(), t[:, 2].long()
    if s.numel() and (int(torch.minimum(s, o).min()) < 0 or int(torch.maximum(s, o).max()) >= n):
        raise ValueError("graph_counts: node ids must be in [0, n_nodes)")
    keys = torch.unique(torch.minimum(s, o) * n + torch.maximum(s, o))  # one key per undirected edge
    a, b = keys // n, keys % n
    degree = torch.bincount(a, minlength=n) + torch.bincount(b, minlength=n)  # a == b: a self-loop counts twice
    a, b = a[a != b], b[a != b]
    src, dst = torch.cat([a, b]), torch.cat([b, a])
    perm = torch.argsort(src * n + dst)
    src, nbr = src[perm], dst[perm].to(torch.int32).contiguous()
    d = torch.bincount(src, minlength=n)
    offsets = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    torch.cumsum(d, 0, out=offsets[1:])
    work = torch.zeros(n, dtype=torch.int64, device=dev).index_add_(0, src, d[nbr.long()])
    order = torch.argsort(work, descending=True).to(torch.int32).contiguous()
    return degree, d, offsets, nbr, order


def graph_counts_csr(offsets, nbr, order):
    """kge_graph_counts on a CSR of graph_csr -> (tri2, sq, pot), int64 [n] on its device, stream-ordered."""
    lib, dev, n = _lib.load(), offsets.device, offsets.numel() - 1
    with torch.cuda.device(dev):
        tri2, sq, pot = (torch.zeros(n, dtype=torch.int64, device=dev) for _ in range(3))
        if nbr.numel() == 0:  # no edge: every count is 0 (and an empty tensor's data pointer is NULL)
            return tri2, sq, pot
        need = int(lib.kge_graph_workspace_bytes(n))
        if n > 0 and need == 0:
            raise RuntimeError("kge_graph_workspace_bytes failed for %d nodes" % n)
        ws = torch.empty(max(need, 8), dtype=torch.uint8, device=dev)
        stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        _lib.check(lib.kge_graph_counts(_ptr(offsets), _ptr(nbr), _ptr(order), n, _ptr(tri2), _ptr(sq), _ptr(pot),
                                        _ptr(ws), need, stream))
    return tri2, sq, pot


def graph_counts(triples, n_nodes, device=None):
    """Per-node statistics of the undirected simple graph of indexed triples (kge_graph_counts, DESIGN.md 3.9).

    triples: [n, 3] ints (a CUDA tensor or a host array); each triple (s, p, o) is an edge {s, o}, s and o in
    [0, n_nodes).  Repeated edges and the two directions of one edge count once; self-loops are left out of the
    adjacency.  device: the CUDA device to run on (default: that of a CUDA `triples`, else the current one).
    Returns a dict of int64 [n_nodes] tensors on that device:
      degree -- nx.Graph.degree (a self-loop counts twice),
      d      -- |N(v)|, the degree without self-loops,
      tri2, sq, pot -- the kernel's counts: nx.triangles = tri2 / 2, nx.clustering = tri2 / (d (d - 1)) (0 if tri2 = 0),
      nx.square_clustering = sq / pot (0 if d < 2 or pot <= 0).
    The CSR is built on the device (graph_csr), then one kge_graph_counts call counts the wedges."""
    degree, d, offsets, nbr, order = graph_csr(triples, n_nodes, device)
    tri2, sq, pot = graph_counts_csr(offsets, nbr, order)
    return {"degree": degree, "d": d, "tri2": tri2, "sq": sq, "pot": pot}


_NVTX = os.environ.get("KGE_B200_NVTX", "0") == "1"


def _traced(name):
    """KGE_B200_NVTX=1: wrap the call in an NVTX range, so that `ncu --nvtx --nvtx-include "kge.train_step/"` (or an
    nsys timeline) attributes kernels to the step phase that launched them.  Off (default): the method is untouched."""
    def deco(fn):
        if not _NVTX:
            return fn

        def wrapped(*a, **k):
            torch.cuda.nvtx.range_push(name)
            try:
                return fn(*a, **k)
            finally:
                torch.cuda.nvtx.range_pop()
        wrapped.__name__, wrapped.__doc__ = fn.__name__, fn.__doc__
        return wrapped
    return deco


class KGEEngine:
    def __init__(self, scoring_type, k, eta, n_ent, n_rel, loss="pairwise", loss_params=None,
                 optimizer="adam", optimizer_params=None, regularizer=None, device=0, neg_group=0,
                 table_alloc=None, ent_rows=None, max_rel_size=None, rank_mode=None, rank_pair_cap=0, lazy_tables=None):
        """regularizer: None | {"p":, "lambda": [, "p2":, "lambda2":]} | {"kind": "N3", "lambda":} | a pair
        [entities, relations] of those (EmbeddingLookupLayer.py:131-155), or {"kind": "DURA", "lambda":, "alpha":,
        "beta":} given for both tables.  An LP term goes to the optimizer; N3 is n3_backward's and DURA
        dura_backward's.  lazy_tables: see set_optimizer.  max_rel_size: RotatE phase normalisation when it differs from the
        relation-table rows (RotatE.py:96).  rank_mode: 'auto' (tensor-core filter + exact refine for the bilinear
        models) | 'exact' (FP32 canonical chain for every pair); env KGE_B200_RANK_MODE overrides the default."""
        self.lib = _lib.load()
        if not torch.cuda.is_available():
            raise RuntimeError("ampligraph_b200 needs a CUDA device (H100, sm_90a); there is no CPU path")
        if scoring_type not in _lib.SCORING:
            raise ValueError("Unknown scoring_type: %r" % (scoring_type,))
        if loss not in _lib.LOSSES:
            raise ValueError("Could not interpret loss identifier: %r" % (loss,))
        lp = dict(loss_params or {})
        reduction = lp.get("reduction", "sum")
        if reduction not in _lib.REDUCTIONS:
            raise AssertionError("Invalid value for reduction!")  # loss_functions.py:95-98
        default_margin = 3.0 if loss == "self_adversarial" else 1.0  # loss_functions.py:23,:29
        self.scoring_type, self.k, self.eta = scoring_type, int(k), int(eta)
        self.n_ent, self.n_rel = int(n_ent), int(n_rel)
        self.reduction = reduction
        # rows of the LOCAL entity table: n_ent, or one row shard of it (parallel.ShardedTrainer)
        self.ent_rows = int(ent_rows) if ent_rows is not None else self.n_ent
        self.device = torch.device("cuda", device)
        cfg = _lib.KgeConfig(C.sizeof(_lib.KgeConfig), _lib.SCORING[scoring_type], int(k), int(eta), int(n_ent),
                             int(n_rel), _lib.LOSSES[loss], _lib.REDUCTIONS[reduction],
                             float(lp.get("margin", default_margin)), float(lp.get("alpha", 0.5)), int(device),
                             int(neg_group), int(max_rel_size or 0),
                             _lib.RANK_MODES[rank_mode or os.environ.get("KGE_B200_RANK_MODE", "auto")], int(rank_pair_cap))
        h = C.c_void_p()
        _lib.check(self.lib.kge_create(C.byref(cfg), C.byref(h)))
        self.h = h
        self.internal_k = self.lib.kge_internal_k(h)
        self.kp = self.lib.kge_half_stride(h)
        self.ld = self.lib.kge_row_stride(h)
        with torch.cuda.device(self.device):
            z = lambda rows: torch.zeros((rows, self.ld), dtype=torch.float32, device=self.device)
            if table_alloc is not None:  # e.g. symmetric (peer-mappable) memory for the multi-GPU path
                self.ent, self.rel, self.g_ent, self.g_rel = table_alloc(self.ent_rows, self.n_rel, self.ld, self.device)
                for t_ in (self.ent, self.rel, self.g_ent, self.g_rel):
                    assert t_.is_contiguous() and t_.dtype == torch.float32
            else:
                # one [ent | rel] block per kind (rows have the same width): the dense optimizer then updates both tables
                # in ONE launch (apply_gradients) -- one launch gap less per step
                self._pblock, self._gblock = z(self.ent_rows + self.n_rel), z(self.ent_rows + self.n_rel)
                self.ent, self.rel = self._pblock[:self.ent_rows], self._pblock[self.ent_rows:]
                self.g_ent, self.g_rel = self._gblock[:self.ent_rows], self._gblock[self.ent_rows:]
            self.loss_acc = torch.zeros(2, dtype=torch.float64, device=self.device)  # [batch loss, reg loss]
        self.set_optimizer(optimizer, optimizer_params, regularizer, lazy_tables)
        self.launches = 0  # kernels launched by this engine (bench.py reports it)
        self._rank_ws = None  # caller-owned ranking workspace (kge_rank_workspace_bytes), grown on demand
        self._pblock_next = None  # second [ent | rel] parameter block of the deferred steps, allocated on first use
        self._deferred = False  # a forward_backward(defer=True) left its replaced-row sum for apply_gradients

    # -- lifetime ---------------------------------------------------------
    def close(self):
        if getattr(self, "h", None) is not None and self.h.value:
            self.lib.kge_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    # -- optimizer state (optimizers.py:255-291) ---------------------------
    def set_optimizer(self, name="adam", params=None, regularizer=None, lazy_tables=None):
        """name: a key of _lib.OPTIMIZERS, or 'lazy_<name>' (extension): update only the rows the step looked up
        (kge_optimizer_step_lazy) in both tables.  lazy_tables: None (the name decides) or a pair (entities, relations)
        of bools that chooses the looked-up-rows rule per table, e.g. the reference's rule for Adamax with a regulariser
        on the entities only (latent_features.optimizers.table_rules)."""
        name = name.lower()
        prefixed = name.startswith("lazy_")
        if prefixed:
            name = name[len("lazy_"):]
        if name not in _lib.OPTIMIZERS:
            raise ValueError("Could not interpret optimizer identifier: %r" % (name,))
        lazy = (prefixed, prefixed) if lazy_tables is None else tuple(bool(x) for x in lazy_tables)
        assert len(lazy) == 2, "Incorrect length for lazy_tables. Expected 2, got {}".format(len(lazy))
        self.lazy_tables = {"ent": lazy[0], "rel": lazy[1]}
        self.lazy = any(lazy)
        p = dict(params or {})
        if name == "rmsprop" and p.get("centered") and float(p.get("momentum", 0.0)) != 0.0:
            raise NotImplementedError("centered RMSprop with momentum needs a third slot buffer (not supported)")
        regs = list(regularizer) if isinstance(regularizer, (list, tuple)) else [regularizer, regularizer]
        assert len(regs) == 2, "Incorrect length for regularizer. Expected 2, got {}".format(len(regs))

        # N3 (DESIGN.md 3.15) is not an optimizer term: its lambdas are n3_backward's, and the optimizer sees no regulariser
        n3 = [float(r["lambda"]) if (r or {}).get("kind") == "N3" else 0.0 for r in regs]
        self.n3_lambdas = {"ent": n3[0], "rel": n3[1]}
        regs = [None if (r or {}).get("kind") == "N3" else r for r in regs]
        # DURA (DESIGN.md 3.16) couples the tables, so it comes as the same config for both; its weights (w_n, w_p) =
        # (lambda alpha, lambda beta), formed in double, are dura_backward's
        dura = [r for r in regs if (r or {}).get("kind") == "DURA"]
        if dura and not (len(dura) == 2 and dura[0] == dura[1]):
            raise ValueError("the DURA regularizer couples the entity and relation tables: give it for both")
        self.dura_weights = None if not dura else (float(dura[0]["lambda"]) * float(dura[0]["alpha"]),
                                                   float(dura[0]["lambda"]) * float(dura[0]["beta"]))
        regs = [None if (r or {}).get("kind") == "DURA" else r for r in regs]

        def cfg_for(reg):
            reg = dict(reg or {})
            return _lib.KgeOptimizerConfig(
                C.sizeof(_lib.KgeOptimizerConfig), _lib.OPTIMIZERS[name], float(p.get("learning_rate", 0.001)),
                float(p.get("beta_1", 0.9)), float(p.get("beta_2", 0.999)), float(p.get("epsilon", 1e-7)),
                float(p.get("momentum", 0.0)), float(p.get("initial_accumulator_value", 0.1)),
                int(reg.get("p", 2)) if reg else 0, float(reg.get("lambda", 1e-5)),
                int(reg.get("p2", 0)) if reg else 0, float(reg.get("lambda2", 0.0)),
                float(p.get("rho", RHO_DEFAULT.get(name, 0.0))), int(bool(p.get("centered", False))))
        self.opt_cfgs = {"ent": cfg_for(regs[0]), "rel": cfg_for(regs[1])}
        self.opt_cfg = self.opt_cfgs["ent"]  # hyper-parameters are common to both tables; only the regulariser differs
        self.opt_name = name
        self.t = 0
        # slots as [ent | rel] blocks, like the tables (see __init__): slots[key] are row slices of them
        mk = lambda v: None if v is None else torch.full((self.ent_rows + self.n_rel, self.ld), v, dtype=torch.float32,
                                                         device=self.device)
        cut = lambda blk: {"ent": None if blk is None else blk[:self.ent_rows], "rel": None if blk is None else blk[self.ent_rows:]}
        b0, b1 = (mk(v) for v in optimizer_slots(self.opt_cfg))
        self._sblocks = (b0, b1)
        self.slots = {key: [cut(b0)[key], cut(b1)[key]] for key in ("ent", "rel")}
        self.stamps = {"ent": None, "rel": None}
        if self.lazy:  # both: the training kernels stamp only while the entity buffer is set
            self.stamps = {"ent": torch.zeros(self.ent_rows, dtype=torch.int32, device=self.device),
                           "rel": torch.zeros(self.n_rel, dtype=torch.int32, device=self.device)}
        _lib.check(self.lib.kge_set_row_stamps(self.h, _ptr(self.stamps["ent"]), _ptr(self.stamps["rel"])))
        self._last_step = 0

    # -- tables ------------------------------------------------------------
    def ensure_row_stash(self, B):
        """Local [B*eta, ld] stash the gradient pass re-reads instead of gathering the replaced rows a second time
        (kge_set_row_stash); a no-op when the kernel keeps every row window resident."""
        if self.lib.kge_rows_resident(self.h) != 0:
            return None
        need = int(B) * self.eta
        if getattr(self, "row_stash", None) is None or self.row_stash.shape[0] < need:
            self.row_stash = torch.empty((need, self.ld), dtype=torch.float32, device=self.device)
            _lib.check(self.lib.kge_set_row_stash(self.h, _ptr(self.row_stash), need))
        return self.row_stash

    def ensure_train_workspace(self, B):
        """The training workspace kge_train_step uses to sum the replaced entities' gradient rows per entity
        (kge_set_train_workspace): one cached buffer, grown with B; nothing where the library's path does not apply.
        Returns whether a fused step of B positives takes that path."""
        need = int(self.lib.kge_train_workspace_bytes(self.h, int(B)))
        if need > 0 and (getattr(self, "_train_ws", None) is None or self._train_ws.numel() < need):
            self._train_ws = torch.empty(need, dtype=torch.uint8, device=self.device)
            _lib.check(self.lib.kge_set_train_workspace(self.h, _ptr(self._train_ws), need, self._stream()))
        return need > 0

    def set_hot_entities(self, triples=None, ids=None):
        """Hot-entity hint (kge_set_hot_entities): the two most frequent subject/object ids of `triples` (numpy / torch
        [N,3] of indexed triples) or explicit `ids`; None/empty clears it."""
        if ids is None and triples is not None:
            t = triples.detach().cpu().numpy() if torch.is_tensor(triples) else np.asarray(triples)
            cnt = np.bincount(np.concatenate([t[:, 0], t[:, 2]]).astype(np.int64), minlength=self.n_ent)
            top = np.argsort(-cnt, kind="stable")[:2]
            ids = [int(e) for e in top if cnt[e] > 0]
        arr = np.asarray(ids if ids is not None else [], dtype=np.int32)
        _lib.check(self.lib.kge_set_hot_entities(self.h, arr.ctypes.data_as(C.c_void_p), int(arr.size)))
        self.hot_entities = arr.tolist()

    def set_embeddings(self, ent_dense=None, rel_dense=None):
        """dense [rows, internal_k] (numpy / torch) -> padded device layout."""
        for dense, table, rows in ((ent_dense, self.ent, self.ent_rows), (rel_dense, self.rel, self.n_rel)):
            if dense is None:
                continue
            d = torch.as_tensor(np.ascontiguousarray(dense, dtype=np.float32) if not torch.is_tensor(dense) else dense)
            d = d.to(self.device, torch.float32).contiguous()
            if tuple(d.shape) != (rows, self.internal_k):
                raise ValueError("expected shape %s, got %s" % ((rows, self.internal_k), tuple(d.shape)))
            _lib.check(self.lib.kge_pack_rows(self.h, _ptr(d), _ptr(table), rows, self._stream()))
            torch.cuda.current_stream(self.device).synchronize()  # d may be freed after return

    def get_embeddings(self):
        out = []
        for table, rows in ((self.ent, self.ent_rows), (self.rel, self.n_rel)):
            d = torch.empty((rows, self.internal_k), dtype=torch.float32, device=self.device)
            _lib.check(self.lib.kge_unpack_rows(self.h, _ptr(table), _ptr(d), rows, self._stream()))
            out.append(d)
        return out[0], out[1]

    def init_glorot_uniform(self, seed=0, only=None):
        if only in (None, "ent"):
            _lib.check(self.lib.kge_init_glorot_uniform(self.h, _ptr(self.ent), self.ent_rows, int(seed) * 2 + 0, self._stream()))
        if only in (None, "rel"):
            _lib.check(self.lib.kge_init_glorot_uniform(self.h, _ptr(self.rel), self.n_rel, int(seed) * 2 + 1, self._stream()))

    def init_table(self, which, kind, a=0.0, b=0.0, seed=0):
        """kge_init_table on the 'ent' or 'rel' table: kind in _lib.INIT_KINDS (uniform [a,b) | normal (mean a, stddev b) |
        truncated_normal | constant a)."""
        table, rows = (self.ent, self.ent_rows) if which == "ent" else (self.rel, self.n_rel)
        _lib.check(self.lib.kge_init_table(self.h, _ptr(table), rows, _lib.INIT_KINDS[kind], float(a), float(b),
                                           int(seed) * 2 + (0 if which == "ent" else 1), self._stream()))

    # -- training ------------------------------------------------------------
    @_traced("kge.train_step")
    def forward_backward(self, triples, negatives=None, seed=0, step=0, mode=_lib.STEP_FUSED,
                         scores_pos=None, scores_neg=None, dpos=None, dneg=None, defer=False):
        """train_step up to tape.gradient: accumulates into g_ent/g_rel and loss_acc[0].

        defer=True (callers that call apply_gradients() next and read nothing in between): where the step sums the
        replaced entities' gradient rows per entity and the dense optimizer takes both tables in one launch, that sum is
        left pending (KGE_STEP_FUSED_DEFER) and apply_gradients() runs it together with the optimizer
        (kge_optimizer_step_deferred); g_ent / g_rel are then incomplete until it does.  The step defers exactly where
        kge_train_workspace_bytes(h, B) > 0 (the library's one decision whether a step buckets); elsewhere defer has no
        effect.  That apply_gradients() writes the new tables to a second block: see its docstring."""
        assert triples.dtype == torch.int32 and triples.is_cuda and triples.is_contiguous()
        if self._deferred:  # its entries live in the training workspace, which this step would overwrite or regrow
            raise ValueError("forward_backward: the replaced-row sum of a deferred step is pending (apply_gradients first)")
        B = triples.shape[0]
        neg_ent = neg_keep = None
        if negatives is not None:
            neg_ent, neg_keep = negatives
            assert neg_ent.dtype == torch.int32 and neg_keep.dtype == torch.uint8
            assert neg_ent.numel() == B * self.eta and neg_keep.numel() == B * self.eta
        bucketed = mode != _lib.STEP_FORWARD_ONLY and self.ensure_train_workspace(B)
        defer = bool(defer) and bucketed and mode == _lib.STEP_FUSED and self._one_block()
        _lib.check(self.lib.kge_train_step(
            self.h, _lib.STEP_FUSED_DEFER if defer else mode, _ptr(self.ent), _ptr(self.rel), _ptr(self.g_ent),
            _ptr(self.g_rel), _ptr(triples), B, _ptr(neg_ent), _ptr(neg_keep), int(seed), int(step), _ptr(self.loss_acc),
            _ptr(scores_pos), _ptr(scores_neg), _ptr(dpos), _ptr(dneg), self._stream()))
        self._deferred = defer
        self._last_step = int(step)
        # RotatE: rotation table + kernel; bucketed: count, two scan launches, kernel, bucket sum (deferred: in
        # apply_gradients' launch)
        self.launches += 2 if self.scoring_type == "RotatE" else (4 if defer else 5) if bucketed else 1

    def _step_call(self, name, fn, need, triples, step, head, tail, pending_ok=False):
        """What the step entry points beside kge_train_step share: check the int32 [B, 3] triples (or queries), refuse
        while a deferred step is pending (unless pending_ok), call fn(h, *head, ent, rel, g_ent, g_rel, triples, B,
        *tail, workspace, need, stream) with the cached scratch of _workspace (the library wants 16-byte alignment;
        every call runs on the engine's stream, so one buffer serves them all in stream order) and keep `step` as the
        lazy optimizer's row stamp.  need=None: the entry point takes no workspace, fn(..., *tail, stream)."""
        assert triples.dtype == torch.int32 and triples.is_cuda and triples.is_contiguous()
        if self._deferred and not pending_ok:
            raise ValueError("%s: the replaced-row sum of a deferred step is pending (apply_gradients first)" % name)
        if need is not None:
            ws, need = self._workspace(int(need))
            tail = tuple(tail) + (_ptr(ws), need)
        _lib.check(fn(self.h, *head, _ptr(self.ent), _ptr(self.rel), _ptr(self.g_ent), _ptr(self.g_rel), _ptr(triples),
                      triples.shape[0], *tail, self._stream()))
        self._last_step = int(step)

    @_traced("kge.one_vs_all_step")
    def one_vs_all_backward(self, triples, sides="s,o", step=0):
        """1vsAll step up to tape.gradient (kge_one_vs_all_step, DESIGN.md 3.12): the multiclass NLL of every positive
        against every entity on each side in `sides` ('s,o', 'o' or 's'), with the engine's reduction; accumulates into
        g_ent / g_rel and loss_acc[0] like forward_backward.  step: the lazy optimizer's row stamp (every entity row and
        the batch's relation rows count as looked up).  apply_gradients() takes its non-deferred path next."""
        if sides not in _lib.ONE_VS_ALL_SIDES:
            raise ValueError("one_vs_all must be one of %s, got %r" % (", ".join(map(repr, _lib.ONE_VS_ALL_SIDES)), sides))
        B = triples.shape[0]
        self._step_call("one_vs_all_backward", self.lib.kge_one_vs_all_step,
                        self.lib.kge_one_vs_all_workspace_bytes(self.h, B), triples, step,
                        (_lib.ONE_VS_ALL_SIDES[sides], _lib.REDUCTIONS[self.reduction]), (int(step), _ptr(self.loss_acc)))
        # query vectors (two kernels), entity stamps, five passes per side
        if B:
            self.launches += 2 + (1 if self.lazy else 0) + 5 * (2 if sides == "s,o" else 1)

    @_traced("kge.one_vs_all_relation_step")
    def one_vs_all_relation_backward(self, triples, weight, step=0):
        """Relation-prediction term of a 1vsAll step up to tape.gradient (kge_one_vs_all_relation_step, DESIGN.md
        3.14): weight * the multiclass NLL of every positive's relation against every relation, scored as f(s, r, o),
        with the engine's reduction; accumulates into g_ent / g_rel and loss_acc[0] like one_vs_all_backward.  step:
        the lazy optimizer's row stamp (every relation row and the batch's s and o rows count as looked up)."""
        B = triples.shape[0]
        self._step_call("one_vs_all_relation_backward", self.lib.kge_one_vs_all_relation_step,
                        self.lib.kge_one_vs_all_relation_workspace_bytes(self.h, B), triples, step,
                        (float(weight), _lib.REDUCTIONS[self.reduction]), (int(step), _ptr(self.loss_acc)))
        # relation stamps, relation queries, five passes, the dX split sum when dX is split
        if B:
            self.launches += (1 if self.lazy else 0) + 6 + (1 if one_vs_all_splits(self.n_rel, B) > 1 else 0)

    @_traced("kge.k_vs_all_step")
    def k_vs_all_backward(self, queries, side, label_offsets, label_ids, label_smoothing=0.0, step=0):
        """KvsAll step up to tape.gradient (kge_k_vs_all_step, DESIGN.md 3.13): the multi-label NLL of every query row
        of `queries` (int32 [B, 3] on the device) against every entity on `side` ('o': (s, p) queries, 's': (p, o)),
        with the engine's reduction and label smoothing eps; accumulates into g_ent / g_rel and loss_acc[0] like
        forward_backward.  The labels of query b are label_ids[label_offsets[b]:label_offsets[b + 1]] (int64 offsets
        [B + 1], absolute into the int32 id array; ascending and distinct per query): a batch is a slice of the
        queries and of the offsets over the same id array.  step: the lazy optimizer's row stamp (every entity row and
        the batch's relation rows count as looked up).  apply_gradients() takes its non-deferred path next."""
        assert label_offsets.dtype == torch.int64 and label_offsets.is_cuda and label_offsets.is_contiguous()
        assert label_ids.dtype == torch.int32 and label_ids.is_cuda and label_ids.is_contiguous()
        if side not in ("s", "o"):
            raise ValueError("k_vs_all_backward: side must be 's' or 'o', got %r" % (side,))
        B = queries.shape[0]
        assert label_offsets.numel() == B + 1
        self._step_call("k_vs_all_backward", self.lib.kge_k_vs_all_step, self.lib.kge_k_vs_all_workspace_bytes(self.h, B),
                        queries, step,
                        (_lib.ONE_VS_ALL_SIDES[side], _lib.REDUCTIONS[self.reduction], float(label_smoothing)),
                        (_ptr(label_offsets), _ptr(label_ids), int(step), _ptr(self.loss_acc)))
        # query vectors (two kernels), entity stamps, dQ, dX and chain
        if B:
            self.launches += 2 + (1 if self.lazy else 0) + 3

    @property
    def n3_workspace_bytes(self):
        """kge_n3_workspace_bytes(h): one int32 count per row of the [ent | rel] block, rounded up to 16 bytes."""
        return (4 * (self.n_ent + self.n_rel) + 15) // 16 * 16

    @_traced("kge.n3_step")
    def n3_backward(self, triples, step=0):
        """The N3 regulariser of a step's positives up to tape.gradient (kge_n3_step, DESIGN.md 3.15): lambda *
        sum_d |z_d|^3 of each positive's s and o rows (entity lambda) and p row (relation lambda), lambdas from the
        engine's regulariser config (n3_lambdas); adds into g_ent / g_rel and loss_acc[1], like the LP term of the
        optimizer.  Call it once per step, after the data term(s) and before apply_gradients().  Allowed while a
        deferred step is pending: the deferred optimizer reads every gradient row.  step: the lazy optimizer's row
        stamp."""
        lam_e, lam_r = self.n3_lambdas["ent"], self.n3_lambdas["rel"]
        if lam_e == 0.0 and lam_r == 0.0:
            raise ValueError("n3_backward: no table of this engine has the N3 regulariser")
        if self.ent_rows != self.n_ent:
            raise NotImplementedError("the N3 regularizer needs the whole entity table: row-sharded tables are not supported")
        self._step_call("n3_backward", self.lib.kge_n3_step, self.n3_workspace_bytes, triples, step, (lam_e, lam_r),
                        (int(step), C.c_void_p(self.loss_acc.data_ptr() + 8)), pending_ok=True)
        if triples.shape[0]:
            self.launches += 2  # count and apply (and a memset)

    @_traced("kge.dura_step")
    def dura_backward(self, triples, step=0):
        """The DURA regulariser of a step's positives up to tape.gradient (kge_dura_step, DESIGN.md 3.16): w_n (|h|^2 +
        |t|^2) + w_p (|h o r|^2 + |t o conj(r)|^2) of each positive, weights from the engine's regulariser config
        (dura_weights); adds into g_ent / g_rel and loss_acc[1], like the LP term of the optimizer.  Call it once per
        step, after the data term(s) and before apply_gradients().  Allowed while a deferred step is pending: the
        deferred optimizer reads every gradient row.  step: the lazy optimizer's row stamp."""
        if self.dura_weights is None:
            raise ValueError("dura_backward: this engine has no DURA regulariser")
        if self.ent_rows != self.n_ent:
            raise NotImplementedError("the DURA regularizer needs the whole entity table: row-sharded tables are not "
                                      "supported")
        w_n, w_p = self.dura_weights
        self._step_call("dura_backward", self.lib.kge_dura_step, None, triples, step, (w_n, w_p),
                        (int(step), C.c_void_p(self.loss_acc.data_ptr() + 8)), pending_ok=True)
        if triples.shape[0]:
            self.launches += 1

    def _one_block(self):
        """True when tables, gradients and slots still ARE the [ent | rel] blocks allocated here (callers may rebind them: the
        multi-GPU trainers do) and both tables share one regulariser: the dense optimizer can take them in one launch."""
        pb, gb = getattr(self, "_pblock", None), getattr(self, "_gblock", None)
        if self.lazy or pb is None:
            return False
        off = self.ent_rows * self.ld * 4

        def is_split(blk, a, b):
            if blk is None:
                return a is None and b is None
            return a is not None and b is not None and a.data_ptr() == blk.data_ptr() and b.data_ptr() == blk.data_ptr() + off

        ce, cr = self.opt_cfgs["ent"], self.opt_cfgs["rel"]
        same_reg = all(getattr(ce, f) == getattr(cr, f) for f, _ in ce._fields_)
        return (same_reg and is_split(pb, self.ent, self.rel) and is_split(gb, self.g_ent, self.g_rel)
                and is_split(self._sblocks[0], self.slots["ent"][0], self.slots["rel"][0])
                and is_split(self._sblocks[1], self.slots["ent"][1], self.slots["rel"][1]))

    @_traced("kge.optimizer_step")
    def apply_gradients(self):
        """optimizer.apply_gradients on both tables (dense semantics) + LP regulariser.

        After a deferred forward_backward the new tables are written to the engine's second parameter block, which then
        becomes the current one: self.ent / self.rel are re-sliced from it, and the block they viewed before is
        overwritten by the next deferred step.  Read self.ent / self.rel (or get_embeddings()) after the step; do not
        hold them across steps."""
        self.t += 1
        if self._deferred:
            # the pending replaced-row sum and the optimizer in one launch: it reads the current block and writes every
            # element of the other one, which becomes the current block (ent / rel are re-sliced from it)
            if self._pblock_next is None:
                self._pblock_next = torch.empty_like(self._pblock)
            rows = self.ent_rows + self.n_rel
            rc = self.lib.kge_optimizer_step_deferred(
                self.h, C.byref(self.opt_cfgs["ent"]), self.t, _ptr(self._pblock), _ptr(self._pblock_next),
                _ptr(self._gblock), _ptr(self._sblocks[0]), _ptr(self._sblocks[1]), rows,
                C.c_void_p(self.loss_acc.data_ptr() + 8), self._stream())
            if rc == _lib.KGE_ERR_INVALID_ARGUMENT:
                self.t -= 1  # arguments refused: nothing ran, and the step stays pending in the library too
            else:
                self._deferred = False  # the library consumed the pending sum, whether or not its launch succeeded
            _lib.check(rc)
            self._pblock, self._pblock_next = self._pblock_next, self._pblock
            self.ent, self.rel = self._pblock[:self.ent_rows], self._pblock[self.ent_rows:]
            self.launches += 1
            return
        if self._one_block():
            _lib.check(self.lib.kge_optimizer_step(
                self.h, C.byref(self.opt_cfgs["ent"]), self.t, _ptr(self._pblock), _ptr(self._gblock), _ptr(self._sblocks[0]),
                _ptr(self._sblocks[1]), self.ent_rows + self.n_rel, C.c_void_p(self.loss_acc.data_ptr() + 8), self._stream()))
            self.launches += 1
            return
        for key, table, grad, rows in (("ent", self.ent, self.g_ent, self.ent_rows),
                                       ("rel", self.rel, self.g_rel, self.n_rel)):
            s0, s1 = self.slots[key]
            if self.lazy_tables[key]:
                _lib.check(self.lib.kge_optimizer_step_lazy(
                    self.h, C.byref(self.opt_cfgs[key]), self.t, _ptr(table), _ptr(grad), _ptr(s0), _ptr(s1), rows,
                    _ptr(self.stamps[key]), self.lib.kge_step_stamp(self._last_step),
                    C.c_void_p(self.loss_acc.data_ptr() + 8), self._stream()))
                continue
            _lib.check(self.lib.kge_optimizer_step(
                self.h, C.byref(self.opt_cfgs[key]), self.t, _ptr(table), _ptr(grad), _ptr(s0), _ptr(s1), rows,
                C.c_void_p(self.loss_acc.data_ptr() + 8), self._stream()))
        self.launches += 2

    def train_step(self, triples, negatives=None, seed=0, step=None):
        """One reference train_step (models/ScoringBasedEmbeddingModel.py:370-429).  Deferred where it can be
        (forward_backward(defer=True)), so self.ent / self.rel may be views of another block afterwards: do not hold them
        across steps (apply_gradients)."""
        self.forward_backward(triples, negatives, seed, self.t if step is None else step, defer=True)
        self.apply_gradients()

    def read_loss(self, reset=True):
        """(batch loss + regulariser loss) accumulated since the last reset; synchronises."""
        v = float(self.loss_acc.cpu().sum())  # one 16-byte D2H copy (synchronising), summed on the host: no reduce kernel
        if reset:
            self.loss_acc.zero_()
        return v

    def generate_corruptions(self, triples, seed=0, step=0):
        out = torch.empty((triples.shape[0] * self.eta, 3), dtype=torch.int32, device=self.device)
        _lib.check(self.lib.kge_generate_corruptions(self.h, _ptr(triples), triples.shape[0], int(seed), int(step),
                                                     _ptr(out), self._stream()))
        return out

    # -- inference -------------------------------------------------------------
    @_traced("kge.score_triples")
    def score(self, triples):
        assert triples.dtype == torch.int32 and triples.is_cuda and triples.is_contiguous()
        out = torch.empty(triples.shape[0], dtype=torch.float32, device=self.device)
        _lib.check(self.lib.kge_score_triples(self.h, _ptr(self.ent), _ptr(self.rel), _ptr(triples), triples.shape[0],
                                              _ptr(out), self._stream()))
        self.launches += 2 if self.scoring_type == "RotatE" else 1
        return out

    def _n_cand(self, side, cand_ids, cand_begin):
        """The default candidate count of a ranking / top-k call: every row from cand_begin on of the table `side`
        replaces from (relation rows for 'p', entity rows otherwise), or the length of cand_ids."""
        if cand_ids is not None:
            return cand_ids.numel()
        return (self.n_rel if side == "p" else self.n_ent) - cand_begin

    def rank_workspace(self, b, n_cand):
        """The caller-owned scratch kge_rank needs (kge_rank_workspace_bytes): one cached torch buffer, grown on demand.
        Growing frees the old buffer through torch's stream-ordered caching allocator, so no synchronisation is needed."""
        return self._workspace(int(self.lib.kge_rank_workspace_bytes(self.h, int(b), int(n_cand))))

    def _workspace(self, need):
        """The cached 1024-byte aligned scratch of rank_workspace, at least `need` bytes; top-k and _step_call share it."""
        if self._rank_ws is None or self._rank_ws.numel() < need:
            raw = torch.empty(max(need, 1024) + 1024, dtype=torch.uint8, device=self.device)
            off = (-raw.data_ptr()) % 1024  # the library wants a 1024-byte aligned base (operand tiles of the tensor-core pass)
            self._rank_ws_raw, self._rank_ws = raw, raw[off:off + max(need, 1024)]
        return self._rank_ws, need

    @_traced("kge.rank")
    def rank(self, triples, side, strategy="worst", filt_off=None, filt_idx=None, cand_ids=None, cand_begin=0,
             n_cand=None, out=None, counts=None):
        """get_ranks for one side ('s', 'o', or 'p': relation prediction, candidates are relation ids / rows).  Default:
        returns/accumulates int32 rank counts in `out` (caller adds 1).
        counts=[b,3] int32: accumulate the RAW counters {greater, equal, filtered} there instead (candidate
        partitions must do this and call finalize_ranks once: 'middle' is not additive over partitions)."""
        assert triples.dtype == torch.int32 and triples.is_cuda and triples.is_contiguous()
        b = triples.shape[0]
        if out is None and counts is None:
            out = torch.zeros(b, dtype=torch.int32, device=self.device)
        if n_cand is None:
            n_cand = self._n_cand(side, cand_ids, cand_begin)
        n_filt = int(filt_idx.numel()) if filt_idx is not None else 0
        ws, ws_bytes = self.rank_workspace(b, n_cand)
        _lib.check(self.lib.kge_rank(self.h, _lib.SIDES[side], _lib.STRATEGIES[strategy], _ptr(self.ent), _ptr(self.rel),
                                     _ptr(triples), b, _ptr(cand_ids), int(cand_begin), int(n_cand), _ptr(filt_off),
                                     _ptr(filt_idx), n_filt, _ptr(out) if counts is None else None, _ptr(counts),
                                     _ptr(ws), ws_bytes, self._stream()))
        self.launches += 5
        return out if counts is None else counts

    def finalize_ranks(self, counts, strategy="worst", out=None):
        """ranks += f_strategy(greater, equal) - filtered, once, from raw counters summed over candidate partitions."""
        b = counts.shape[0]
        if out is None:
            out = torch.zeros(b, dtype=torch.int32, device=self.device)
        _lib.check(self.lib.kge_rank_finalize(self.h, _ptr(counts), b, _lib.STRATEGIES[strategy], _ptr(out), self._stream()))
        self.launches += 1
        return out

    def rank_filter_probe(self, triples, side, cand_ids=None, cand_begin=0, n_cand=None):
        """Diagnostic (kge_rank_filter_probe): (approximate tensor-core scores, assumed error bound), both [b, n_cand].
        The bound is NaN for every pair of a query or 256-candidate tile with a NaN or inf entry: the filter refines
        all of them exactly."""
        b = triples.shape[0]
        if n_cand is None:
            n_cand = self._n_cand(side, cand_ids, cand_begin)
        approx = torch.empty((b, int(n_cand)), dtype=torch.float32, device=self.device)
        delta = torch.empty_like(approx)
        ws, ws_bytes = self.rank_workspace(b, n_cand)
        _lib.check(self.lib.kge_rank_filter_probe(self.h, _lib.SIDES[side], _ptr(self.ent), _ptr(self.rel), _ptr(triples), b,
                                                  _ptr(cand_ids), int(cand_begin), int(n_cand), _ptr(approx), _ptr(delta),
                                                  _ptr(ws), ws_bytes, self._stream()))
        return approx, delta

    def corruption_scores(self, triples, side, cand_ids=None, cand_begin=0, n_cand=None):
        """_get_subject_corruption_scores / _get_object_corruption_scores: fp32 [b, n_cand], canonical summation order."""
        assert triples.dtype == torch.int32 and triples.is_cuda and triples.is_contiguous()
        b = triples.shape[0]
        if n_cand is None:
            n_cand = self._n_cand(side, cand_ids, cand_begin)
        out = torch.empty((b, int(n_cand)), dtype=torch.float32, device=self.device)
        ws, ws_bytes = self.rank_workspace(b, n_cand)
        _lib.check(self.lib.kge_corruption_scores(self.h, _lib.SIDES[side], _ptr(self.ent), _ptr(self.rel), _ptr(triples), b,
                                                  _ptr(cand_ids), int(cand_begin), int(n_cand), _ptr(out), _ptr(ws), ws_bytes,
                                                  self._stream()))
        self.launches += 3
        return out

    @_traced("kge.topk")
    def topk(self, triples, side, k, filt_off=None, filt_idx=None, cand_ids=None, cand_begin=0, n_cand=None):
        """Link prediction (kge_topk): the k best candidates on `side` of each query -> (ids int32 [b,k], scores fp32 [b,k])
        on the device, sorted by (score desc, candidate position asc), NaN first; scores bit-identical to
        corruption_scores.  Candidates and filter (candidate positions to exclude) as in rank; rows with fewer than k
        eligible candidates end in id -1 / score -inf."""
        assert triples.dtype == torch.int32 and triples.is_cuda and triples.is_contiguous()
        b = triples.shape[0]
        if n_cand is None:
            n_cand = self._n_cand(side, cand_ids, cand_begin)
        n_filt = int(filt_idx.numel()) if filt_idx is not None else 0
        ids = torch.empty((b, max(int(k), 0)), dtype=torch.int32, device=self.device)
        scores = torch.empty((b, max(int(k), 0)), dtype=torch.float32, device=self.device)
        ws, ws_bytes = self._topk_workspace(self.lib.kge_topk_workspace_bytes(self.h, b, int(n_cand), int(k)))
        _lib.check(self.lib.kge_topk(self.h, _lib.SIDES[side], _ptr(self.ent), _ptr(self.rel), _ptr(triples), b,
                                     _ptr(cand_ids), int(cand_begin), int(n_cand), _ptr(filt_off), _ptr(filt_idx), n_filt,
                                     int(k), _ptr(ids), _ptr(scores), _ptr(ws), ws_bytes, self._stream()))
        return ids, scores

    @_traced("kge.select_topk")
    def select_topk(self, scores, k):
        """kge_select_topk on a [b, n] fp32 device matrix -> (positions int32 [b,k], values fp32 [b,k]), same order and
        padding (-1 / -inf) as topk."""
        assert scores.dtype == torch.float32 and scores.is_cuda and scores.is_contiguous() and scores.dim() == 2
        b, n = scores.shape
        pos = torch.empty((b, max(int(k), 0)), dtype=torch.int32, device=self.device)
        out = torch.empty((b, max(int(k), 0)), dtype=torch.float32, device=self.device)
        ws, ws_bytes = self._topk_workspace(self.lib.kge_select_topk_workspace_bytes(self.h, b, n, int(k)))
        _lib.check(self.lib.kge_select_topk(self.h, _ptr(scores), b, n, int(k), _ptr(pos), _ptr(out), _ptr(ws), ws_bytes,
                                            self._stream()))
        return pos, out

    @_traced("kge.knn")
    def knn(self, points, query_ids, k, metric, cand_ids=None, cand_begin=0, n_cand=None, filt_off=None, filt_idx=None,
            farthest=False):
        """Nearest-neighbour search (kge_knn) over the rows of `points`, any [n, ld] fp32 CUDA tensor with ld % 4 == 0
        (self.ent, self.rel or a gathered matrix): the k nearest (farthest=True: farthest) candidate rows of each row
        query_ids[i] -> (ids int32 [b,k], distances fp32 [b,k]) on the device, distance ascending (farthest:
        descending), ties by candidate position ascending; rows with fewer than k eligible candidates end in id -1 /
        distance +inf (farthest: -inf).  metric: 'euclidean' | 'manhattan'.  Candidates and filter (candidate positions to
        exclude) as in topk."""
        assert points.dtype == torch.float32 and points.is_cuda and points.is_contiguous() and points.dim() == 2
        assert query_ids.dtype == torch.int32 and query_ids.is_cuda and query_ids.is_contiguous()
        b, (n_points, ld) = query_ids.numel(), points.shape
        if n_cand is None:
            n_cand = cand_ids.numel() if cand_ids is not None else n_points - cand_begin
        n_filt = int(filt_idx.numel()) if filt_idx is not None else 0
        ids = torch.empty((b, max(int(k), 0)), dtype=torch.int32, device=self.device)
        dist = torch.empty((b, max(int(k), 0)), dtype=torch.float32, device=self.device)
        ws, ws_bytes = self._topk_workspace(self.lib.kge_knn_workspace_bytes(self.h, b, int(n_cand), int(k), ld))
        _lib.check(self.lib.kge_knn(self.h, _metric(metric), _ptr(points), n_points, ld, _ptr(query_ids), b, _ptr(cand_ids),
                                    int(cand_begin), int(n_cand), _ptr(filt_off), _ptr(filt_idx), n_filt, int(k),
                                    int(bool(farthest)), _ptr(ids), _ptr(dist), _ptr(ws), ws_bytes, self._stream()))
        return ids, dist

    @_traced("kge.radius_neighbors")
    def radius_neighbors(self, points, query_ids, radius, metric, cand_ids=None, cand_begin=0, n_cand=None):
        """Radius search (kge_radius_neighbors): for each row query_ids[i] of `points`, every candidate row at distance
        d <= radius -> (offsets int64 [b+1], ids int32 [offsets[-1]]) on the device, row i's ids in ascending candidate
        position.  d is knn's fp32 distance; radius is taken as the largest fp32 not above it, so the test is exactly
        d <= radius for the Python number.  Two passes (count, then emit into the CSR); synchronises once for the size."""
        head, tail = self._radius_args(points, query_ids, radius, metric, cand_ids, cand_begin, n_cand)
        offsets = torch.zeros(query_ids.numel() + 1, dtype=torch.int64, device=self.device)

        def call(nbr):
            _lib.check(self.lib.kge_radius_neighbors(*head, _ptr(offsets), _ptr(nbr), *tail))
        call(None)
        torch.cumsum(offsets, 0, out=offsets)
        nbr = torch.empty(int(offsets[-1]), dtype=torch.int32, device=self.device)
        if nbr.numel() > 0:  # an empty tensor's data pointer is NULL, which would ask for another count pass
            call(nbr)
        return offsets, nbr

    def _radius_args(self, points, query_ids, radius, metric, cand_ids, cand_begin, n_cand):
        """The leading arguments of the kge_radius_* calls (radius as the largest fp32 not above it) and the trailing
        ones (their workspace, the stream)."""
        assert points.dtype == torch.float32 and points.is_cuda and points.is_contiguous() and points.dim() == 2
        assert query_ids.dtype == torch.int32 and query_ids.is_cuda and query_ids.is_contiguous()
        b, (n_points, ld) = query_ids.numel(), points.shape
        if n_cand is None:
            n_cand = cand_ids.numel() if cand_ids is not None else n_points - cand_begin
        ws, ws_bytes = self._topk_workspace(self.lib.kge_radius_workspace_bytes(self.h, b, int(n_cand), ld))
        head = (self.h, _metric(metric), _ptr(points), n_points, ld, _ptr(query_ids), b, _ptr(cand_ids), int(cand_begin),
                int(n_cand), fp32_floor(radius))
        return head, (_ptr(ws), ws_bytes, self._stream())

    def radius_counts(self, points, query_ids, radius, metric, cand_ids=None, cand_begin=0, n_cand=None):
        """The count pass of radius_neighbors alone: #{candidates at d <= radius} of each query -> int64 [b] on the
        device, without synchronising."""
        head, tail = self._radius_args(points, query_ids, radius, metric, cand_ids, cand_begin, n_cand)
        offsets = torch.zeros(query_ids.numel() + 1, dtype=torch.int64, device=self.device)
        _lib.check(self.lib.kge_radius_neighbors(*head, _ptr(offsets), None, *tail))
        return offsets[1:]

    def radius_union(self, points, query_ids, radius, metric, parent, cand_ids=None, cand_begin=0, n_cand=None):
        """kge_radius_union: joins each row query_ids[i] with every candidate row at d <= radius (radius_neighbors'
        test) in the union-find forest `parent` (int32 [len(points)], parent[x] = x before the first call); a root
        always hooks under the smaller root, so each tree's root is its smallest id."""
        assert parent.dtype == torch.int32 and parent.is_cuda and parent.numel() == points.shape[0]
        head, tail = self._radius_args(points, query_ids, radius, metric, cand_ids, cand_begin, n_cand)
        _lib.check(self.lib.kge_radius_union(*head, _ptr(parent), *tail))

    def radius_min_key(self, points, query_ids, radius, metric, key, cand_ids=None, cand_begin=0, n_cand=None):
        """kge_radius_min_key: the smallest key[c] over the candidate ids c at d <= radius of each row query_ids[i] ->
        int32 [b] on the device, 2^31 - 1 where there is none.  key: int32 [len(points)], indexed by id."""
        assert key.dtype == torch.int32 and key.is_cuda and key.numel() == points.shape[0]
        head, tail = self._radius_args(points, query_ids, radius, metric, cand_ids, cand_begin, n_cand)
        out = torch.empty(query_ids.numel(), dtype=torch.int32, device=self.device)
        _lib.check(self.lib.kge_radius_min_key(*head, _ptr(key), _ptr(out), *tail))
        return out

    def forest_flatten(self, parent):
        """kge_forest_flatten: parent[x] = root(x) for every x, in place, after the unions."""
        assert parent.dtype == torch.int32 and parent.is_cuda and parent.is_contiguous()
        _lib.check(self.lib.kge_forest_flatten(self.h, _ptr(parent), parent.numel(), self._stream()))

    @_traced("kge.dbscan")
    def dbscan(self, points, eps, min_samples, metric, batch=DBSCAN_BATCH):
        """sklearn DBSCAN(eps, min_samples, metric).fit_predict over the rows of `points` (any [n, ld] fp32 CUDA tensor
        with ld % 4 == 0, as for knn), with knn's fp32 distances and the test d <= eps (eps taken as the largest fp32 not
        above it) -> (labels int64 [n], core bool [n]) on the device.  Labels follow sklearn's: clusters numbered by
        their smallest core row, noise -1 (DESIGN.md 3.8).

        Four sweeps of `batch` queries each: the radius count of every row (core: count >= min_samples), the union of
        the in-radius core pairs (queries core[s:e], candidates core[s:], so each pair is scored at most twice), the
        flatten of the forest, and the smallest root among the core neighbours of every non-core row.  Synchronises
        once, to compact the core ids."""
        assert points.dtype == torch.float32 and points.is_cuda and points.is_contiguous() and points.dim() == 2
        n = points.shape[0]
        if not float(eps) > 0:
            raise ValueError("eps must be > 0, got %r" % (eps,))
        if int(min_samples) < 1:
            raise ValueError("min_samples must be >= 1, got %r" % (min_samples,))
        if n >= 2 ** 31:
            raise ValueError("dbscan: ids are int32 (n < 2^31), got n = %d" % n)
        radius, dev = fp32_floor(eps), self.device
        every = torch.arange(n, dtype=torch.int32, device=dev)
        counts = torch.empty(n, dtype=torch.int64, device=dev)
        for s in range(0, n, batch):
            counts[s:s + batch] = self.radius_counts(points, every[s:s + batch], radius, metric, n_cand=n)
        core = counts >= int(min_samples)
        core_ids = torch.nonzero(core).flatten().to(torch.int32)
        parent = every.clone()
        for s in range(0, core_ids.numel(), batch):
            self.radius_union(points, core_ids[s:s + batch], radius, metric, parent, cand_ids=core_ids[s:])
        self.forest_flatten(parent)
        border = torch.full((n,), INT32_MAX, dtype=torch.int32, device=dev)
        if core_ids.numel() > 0:
            rest = torch.nonzero(~core).flatten().to(torch.int32)
            for s in range(0, rest.numel(), batch):
                q = rest[s:s + batch]
                border[q.long()] = self.radius_min_key(points, q, radius, metric, parent, cand_ids=core_ids)
        return dbscan_labels(core, parent, border), core

    def _topk_workspace(self, need):
        # need == 0: invalid arguments (k < 1, ...) -- the call itself reports them
        need = int(need)
        return self._workspace(need) if need > 0 else (None, 0)
