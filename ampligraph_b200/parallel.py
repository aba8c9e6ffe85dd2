"""Multi-GPU host logic: one process per GPU (torch.distributed for the plumbing), peer memory for the data path.

The training path shards naturally over positives (SURVEY.md 8e): every rank runs the fused
kernel on its own slice of the global batch into its own gradient tables, the tables are
summed with ONE exchange (the loss is a SUM over the batch, loss_functions.py:214, so the
summed gradient equals the single-GPU gradient of the global batch), and every rank ends up
with the identical dense optimizer step.  Ranking shards over entity rows: each rank
counts against its row range and the int32 raw counters are summed (rank counts are additive over
entity partitions, ScoringBasedEmbeddingModel.py:1449-1452).
"""
import os

import torch
import torch.distributed as dist


def batch_slot(step, world, rank, n_batches):
    """Which sequential batch of the epoch rank `rank` trains at global step `step`
    (rank-major interleave keeps the reference's sequential order across the job)."""
    return (step * world + rank) % n_batches


def row_shard(n_rows, world, rank):
    """Contiguous row range [begin, end) of rank `rank` (NVSwitch is uniform: no topology awareness)."""
    per = (n_rows + world - 1) // world
    lo = min(rank * per, n_rows)
    return lo, min(lo + per, n_rows)


def allreduce_sum_(tensors, group=None):
    """In-place SUM all-reduce of the gradient tables / rank counters (NCCL on GPUs, gloo in CPU tests)."""
    if not dist.is_available() or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return tensors
    for t in tensors:
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)
    return tensors


def reject_lazy(optimizer_name, world):
    """The lazy (touched-rows-only) optimizer is defined for ONE writer of the row stamps.  With replicated tables every
    rank stamps only the rows of its own batch slice, so a lazy update after the gradient exchange would skip rows other
    ranks touched (ADVICE r1): refuse instead of silently diverging.  Row-sharded tables (ShardedTrainer) do support it --
    there every rank stamps the owner's shard through peer memory."""
    if world > 1 and str(optimizer_name).lower().startswith("lazy_"):
        raise NotImplementedError("optimizer %r with replicated tables on %d GPUs: the lazy rule needs row-sharded tables "
                                  "(parallel.ShardedTrainer); use the dense optimizer for data-parallel training"
                                  % (optimizer_name, world))


def tables_close(got, ref, init, rtol=3e-4, atol_of_update=2e-3, outlier_of_update=5e-2, outlier_fraction=1e-4):
    """Parity criterion for two runs that sum the same fp32 gradient contributions in a different order (multi-GPU vs
    single GPU).  Adam turns a relative gradient difference d into an update difference of about lr*d whatever the size of
    the parameter, so the absolute tolerance is stated relative to how far the parameters MOVED (u = max|ref - init|):
      * all but a fraction `outlier_fraction` of the elements: |got - ref| <= atol_of_update*u + rtol*|ref|;
      * EVERY element: |got - ref| <= outlier_of_update*u + rtol*|ref| -- an element whose summed gradient cancels to ~0 has
        its Adam direction decided by rounding noise (measured before the H100 port: up to 6e-3 u on cfg4 over 8 shards, loss equal to 1e-11),
        whereas a lost or doubled contribution moves a whole row by O(1) u and fails this bound.
    Returns (ok, max_abs_err / u)."""
    import numpy as np
    got, ref, init = (np.asarray(x, dtype=np.float64) for x in (got, ref, init))
    upd = max(float(np.abs(ref - init).max()), 1e-30)
    err = np.abs(got - ref)
    slack = rtol * np.abs(ref)
    tight = err <= atol_of_update * upd + slack
    loose = err <= outlier_of_update * upd + slack
    ok = bool(loose.all()) and float((~tight).mean()) <= outlier_fraction
    return ok, float(err.max() / upd)


_FLAG_WORDS = 64  # uint32 words reserved per rank for the in-kernel barriers (2 slots x up to 8 writers, padded)


class DataParallelTrainer:
    """Replicated tables, one rank per GPU, the reference's train_step on the GLOBAL batch.

    Each rank runs the fused kernel on its own slice of the batch into its own gradient block.
    Preferred path ("p2p"): parameter block [ent|rel], two gradient blocks and a flag pad live in one torch
    symmetric-memory buffer, so every rank can address every peer's copy through NVLink.  The whole tail of the step is
    ONE kernel (kge_optimizer_step_exchange): flag barrier, gradient reduce-scatter by peer loads, the optimizer on this
    rank's row shard (slots are sharded: 1/N of the Adam state per GPU), parameter all-gather by peer stores, flag
    barrier.  Gradient blocks are double-buffered (step i scatters into block i&1 and the exchange zeroes the other
    one), so there is no memset either: 2 launches per step (train kernel + exchange) at any N.
    "nvls" (opt-in, KGE_B200_DP_MODE=nvls): the same kernel, but the gradient shard is reduced inside the NVSwitch
    (multimem.ld_reduce on the multicast mapping) and the new rows are broadcast by it (multimem.st).
    Fallback ("nccl"): SUM all-reduce of the gradient tables + the full optimizer on every replica.
    Both equal the single-GPU step on the concatenated batch up to fp32 summation order, because
    the loss is a SUM over the batch (loss_functions.py:214).
    """

    def __init__(self, make_engine, mode="auto", group=None):
        import ctypes as C
        from . import _lib
        self._C, self._lib = C, _lib
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.mode = "single" if self.world == 1 else mode
        self.hdl = None
        self._k = 0  # exchanges done (gradient block parity, barrier token)
        self._mc = None
        if self.mode in ("auto", "p2p", "nvls"):
            try:
                self.eng = make_engine(self._symmetric_alloc)
                reject_lazy("lazy_" if self.eng.lazy else "", self.world)
                self._finish_p2p_setup()
                # NVLS moves 2/N of a block per rank per step through the links instead of 2(N-1)/N: it wins from 4 GPUs up;
                # at N = 2 the switch round trip of the local contribution makes it slower than p2p
                want_nvls = mode == "nvls" or (mode == "auto" and self.world >= int(os.environ.get("KGE_B200_NVLS_MIN_WORLD", "4")))
                mc = int(getattr(self.hdl, "multicast_ptr", 0) or 0) if want_nvls else 0
                if mode == "nvls" and not mc:
                    raise RuntimeError("symmetric memory has no multicast mapping on this system (NVLS unavailable)")
                if mc:
                    ld = self.eng.ld
                    self._mc = {k: mc + self._row_off[k] * ld * 4 for k in ("table", "g0", "g1")}
                self.mode = "nvls" if mc else "p2p"
            except NotImplementedError:
                raise
            except Exception as e:  # no symmetric memory / no peer access: NCCL path
                if mode in ("p2p", "nvls"):
                    raise
                self.p2p_error = repr(e)
                self.mode = "nccl"
                self.hdl = None
                self.eng = make_engine(None)
        else:
            self.eng = make_engine(None)
        reject_lazy("lazy_" if self.eng.lazy else "", self.world)

    # ---- symmetric-memory plumbing ------------------------------------------------
    def _symmetric_alloc(self, n_ent, n_rel, ld, device):
        """One symmetric buffer [ent | rel | gA_ent | gA_rel | gB_ent | gB_rel | flags] so a single rendezvous maps it all."""
        import torch.distributed._symmetric_memory as symm_mem
        blk = n_ent + n_rel
        flag_rows = (_FLAG_WORDS + ld - 1) // ld
        self._buf = symm_mem.empty((3 * blk + flag_rows, ld), dtype=torch.float32, device=device)
        self._buf.zero_()
        pg = self.group if self.group is not None else dist.group.WORLD
        self.hdl = symm_mem.rendezvous(self._buf, pg.group_name)
        b = self._buf
        self._blk = blk
        self._row_off = {"table": 0, "g0": blk, "g1": 2 * blk, "flags": 3 * blk}
        self._gviews = [(b[blk:blk + n_ent], b[blk + n_ent:2 * blk]), (b[2 * blk:2 * blk + n_ent], b[2 * blk + n_ent:3 * blk])]
        return b[0:n_ent], b[n_ent:blk], self._gviews[0][0], self._gviews[0][1]

    def _finish_p2p_setup(self):
        C, eng = self._C, self.eng
        ld = eng.ld
        base = [int(p) for p in self.hdl.buffer_ptrs]
        assert len(base) == self.world and base[self.rank] == self._buf.data_ptr()
        mk = lambda key: (C.c_void_p * self.world)(*[b + self._row_off[key] * ld * 4 for b in base])
        self._ptrs = {k: mk(k) for k in ("table", "g0", "g1", "flags")}
        self._local_g = [base[self.rank] + self._row_off[k] * ld * 4 for k in ("g0", "g1")]
        self.shard = row_shard(self._blk, self.world, self.rank)  # over the concatenated [ent|rel] rows
        lo, hi = self.shard
        # optimizer slots only for this rank's row shard of the concatenated block
        rows = hi - lo
        from .engine import optimizer_slots
        self.slots = [None if v is None else torch.full((max(rows, 1), ld), v, dtype=torch.float32, device=eng.device)
                      for v in optimizer_slots(eng.opt_cfg)]
        eng.slots = {"ent": [None, None], "rel": [None, None]}  # the full-size slots are not used on this path
        torch.cuda.synchronize()
        self.hdl.barrier(channel=0)  # one-off: every rank's buffer (zeroed flags included) exists before the first step

    # ---- one global step ------------------------------------------------------------
    def train_step(self, batch, negatives=None, seed=0, step=0, kernel_done=None):
        eng = self.eng
        if self.mode in ("p2p", "nvls"):
            blk = self._k & 1
            eng.g_ent, eng.g_rel = self._gviews[blk]
        # one GPU: the replaced-row sum runs inside the optimizer launch (KGEEngine.forward_backward(defer=True))
        eng.forward_backward(batch, negatives, seed=seed, step=step, defer=self.mode == "single")
        if kernel_done is not None:
            kernel_done.record()  # CUDA event: lets bench.py time the fused kernel alone
        if self.mode == "single":
            eng.apply_gradients()
        elif self.mode == "nccl":
            allreduce_sum_([eng.g_ent, eng.g_rel], self.group)
            eng.apply_gradients()
        else:
            C, _lib = self._C, self._lib
            eng.begin_step()
            self._k += 1
            lo, hi = self.shard
            s0, s1 = self.slots
            p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)
            _lib.check(eng.lib.kge_optimizer_step_exchange(
                eng.h, C.byref(eng.opt_cfgs["ent"]), C.byref(eng.opt_cfgs["rel"]), eng.t, self.world, self.rank,
                self._ptrs["table"], self._ptrs["g%d" % blk],
                C.c_void_p(self._mc["table"] if self._mc else 0), C.c_void_p(self._mc["g%d" % blk] if self._mc else 0),
                C.c_void_p(self._local_g[blk ^ 1]), p(s0), p(s1), lo, hi,
                self._ptrs["flags"], self._k, 3, C.c_void_p(eng.loss_acc.data_ptr() + 8), eng._stream()))
            eng.launches += 1

    def trace_exchange(self, on=True):
        """Switch the phase stamps of the exchange kernel on/off (kge_set_exchange_trace); read them with
        exchange_phases_us() after a synchronised step."""
        C = self._C
        self._trace = torch.zeros(8, dtype=torch.int64, device=self.eng.device) if on else None
        self._lib.check(self.eng.lib.kge_set_exchange_trace(self.eng.h, C.c_void_p(self._trace.data_ptr() if on else 0)))

    def exchange_phases_us(self):
        """-> dict of the last exchange launch's phase durations in microseconds (needs trace_exchange(True))."""
        t = self._trace.cpu().tolist()
        d = lambda a, b: (t[b] - t[a]) / 1e3
        return {"zero_next_gradient_block": d(0, 1), "entry_barrier_wait": d(1, 2), "reduce_scatter_optimizer_all_gather": d(2, 3),
                "cta0_fence_and_report": d(3, 4), "wait_for_last_cta": d(4, 5), "exit_flag_exchange": d(5, 6), "kernel_total": d(0, 6)}

    def reduce_loss_(self):
        """SUM the [batch loss, regulariser loss] accumulators over ranks (for logging).  p2p: every rank holds its shard of
        the regulariser loss; nccl: every replica computed the FULL regulariser loss, so it is divided by world first."""
        if self.world > 1:
            if self.mode == "nccl":
                self.eng.loss_acc[1] /= self.world
            dist.all_reduce(self.eng.loss_acc, group=self.group)
        return self.eng.loss_acc

    def close(self):
        self.eng.close()


class ShardedTrainer:
    """Row-sharded entity table (BASELINE configs[3],[4]: tables too large for one GPU).

    Rank r owns entity rows [r*rps, (r+1)*rps) -- table, gradient accumulator and optimizer slots --
    in torch symmetric memory; relations are replicated.  One step of the reference's train_step on
    the GLOBAL batch (each rank feeds its own slice):
      1. kge_train_step_sharded: the fused kernel gathers the rows it needs from whichever rank owns
         them and scatter-adds gradient rows back, all over NVLink peer memory (the forward row
         all-to-all and backward gradient all-to-all of SURVEY.md 8e, fused into the kernel);
      2. flag barrier (kge_peer_barrier); each rank runs the optimizer on its own shard (no exchange), and the
         replicated relation table goes through kge_optimizer_step_sharded (peer reduce + all-gather);
      3. flag barrier.
    This replaces the reference's bucket partitioning through disk (datasets/partitioned_data_manager.py:573-955).
    """

    def __init__(self, scoring_type, k, eta, n_ent, n_rel, device, group=None, lazy=False, **engine_kw):
        """lazy=True: each rank updates only the rows of its shard that the step touched
        (kge_optimizer_step_lazy; opt-in, not the reference's dense rule) -- what makes a 10 M-entity
        table trainable: the dense pass would stream the whole 10 GB shard 8 times per step."""
        import ctypes as C
        import torch.distributed._symmetric_memory as symm_mem
        from . import _lib
        from .engine import KGEEngine
        self._C, self._lib = C, _lib
        self.group = group
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        self.n_ent, self.n_rel = int(n_ent), int(n_rel)
        self.rps = (self.n_ent + self.world - 1) // self.world
        self.first = self.rank * self.rps
        self.n_local = max(0, min(self.rps, self.n_ent - self.first))

        self.lazy = bool(lazy)
        self.use_stash = os.environ.get("KGE_B200_STASH", "1") != "0"
        self._k = 0

        def alloc(rows, n_rel_, ld, dev):
            assert rows == self.rps
            self._stamp_rows = (rows + ld - 1) // ld  # int32 row stamps live in the same symmetric buffer
            flag_rows = (_FLAG_WORDS + ld - 1) // ld
            total = 2 * rows + 2 * n_rel_ + self._stamp_rows + flag_rows
            self._buf = symm_mem.empty((total, ld), dtype=torch.float32, device=dev)
            self._buf.zero_()
            pg = group if group is not None else dist.group.WORLD
            self.hdl = symm_mem.rendezvous(self._buf, pg.group_name)
            self._off = {"ent": 0, "g_ent": rows, "rel": 2 * rows, "g_rel": 2 * rows + n_rel_,
                         "stamp": 2 * rows + 2 * n_rel_, "flags": 2 * rows + 2 * n_rel_ + self._stamp_rows}
            b = self._buf
            return b[0:rows], b[2 * rows:2 * rows + n_rel_], b[rows:2 * rows], b[2 * rows + n_rel_:2 * rows + 2 * n_rel_]

        # the engine itself runs the DENSE rule's bookkeeping (no engine-owned stamps): the entity stamps of a sharded run
        # live in the symmetric buffer so that peers can stamp the owner's rows; optimizer="lazy_adam" implies lazy=True
        opt_name = str(engine_kw.get("optimizer", "adam")).lower()
        if opt_name.startswith("lazy_"):
            self.lazy = True
            engine_kw["optimizer"] = opt_name[len("lazy_"):]
        self.eng = KGEEngine(scoring_type, k, eta, n_ent, n_rel, device=device, table_alloc=alloc, ent_rows=self.rps,
                             **engine_kw)
        eng, ld = self.eng, self.eng.ld
        base = [int(p) for p in self.hdl.buffer_ptrs]
        ptr = lambda q, key: base[q] + self._off[key] * ld * 4
        self.map = _lib.KgeShardMap(C.sizeof(_lib.KgeShardMap), self.world, self.rps)
        for q in range(self.world):
            self.map.ent[q] = ptr(q, "ent")
            self.map.grad_ent[q] = ptr(q, "g_ent")
            self.map.stamp_ent[q] = ptr(q, "stamp") if self.lazy else None
        so = self._off["stamp"]
        self._stamps = self._buf[so:so + self._stamp_rows].view(torch.int32).reshape(-1)[:self.rps]
        self._rel_ptrs = (C.c_void_p * self.world)(*[ptr(q, "rel") for q in range(self.world)])
        self._grel_ptrs = (C.c_void_p * self.world)(*[ptr(q, "g_rel") for q in range(self.world)])
        self._flag_ptrs = (C.c_void_p * self.world)(*[ptr(q, "flags") for q in range(self.world)])
        self.rel_shard = row_shard(self.n_rel, self.world, self.rank)
        lo, hi = self.rel_shard
        eng.slots["rel"] = [None if s is None else s[lo:hi].clone() for s in eng.slots["rel"]]
        torch.cuda.synchronize()
        self.hdl.barrier(channel=0)  # one-off: all buffers exist and are zeroed before the first peer access

    def barrier(self, slot=0):
        """Stream-ordered cross-rank barrier over the flag pad (one 32-thread kernel)."""
        self._k += 1
        self._lib.check(self.eng.lib.kge_peer_barrier(self.eng.h, self.world, self.rank, self._flag_ptrs, int(slot), self._k,
                                                      self.eng._stream()))

    def set_embeddings(self, ent_dense=None, rel_dense=None):
        """dense GLOBAL tables (numpy, identical on every rank): each rank keeps its row slice."""
        import numpy as np
        if ent_dense is not None:
            loc = np.zeros((self.rps, ent_dense.shape[1]), np.float32)
            loc[:self.n_local] = ent_dense[self.first:self.first + self.n_local]
            self.eng.set_embeddings(loc, None)
        if rel_dense is not None:
            self.eng.set_embeddings(None, rel_dense)
        self.barrier(0)

    def get_embeddings(self):
        """-> (global entity table [n_ent, K] gathered from all shards, relation table), torch cpu."""
        ent, rel = self.eng.get_embeddings()
        parts = [torch.empty_like(ent) for _ in range(self.world)]
        dist.all_gather(parts, ent.contiguous(), group=self.group)
        return torch.cat(parts)[:self.n_ent].cpu(), rel.cpu()

    def train_step(self, batch, negatives=None, seed=0, step=0, events=None):
        """events: optional list; receives 5 CUDA events (start, kernel done, barrier 0 done, optimizers done,
        barrier 1 done) so a benchmark can attribute the step time."""
        C, _lib, eng = self._C, self._lib, self.eng
        B = batch.shape[0]
        if self.use_stash:
            eng.ensure_row_stash(B)
        def mark():
            if events is not None:
                e = torch.cuda.Event(enable_timing=True)
                e.record()
                events.append(e)
        mark()
        neg_ent = neg_keep = None
        if negatives is not None:
            neg_ent, neg_keep = negatives
        p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)
        st = eng._stream()
        _lib.check(eng.lib.kge_train_step_sharded(
            eng.h, _lib.STEP_FUSED, C.byref(self.map), p(eng.rel), p(eng.g_rel), p(batch), B, p(neg_ent), p(neg_keep),
            int(seed), int(step), p(eng.loss_acc), None, None, None, None, st))
        mark()
        self.barrier(0)  # every rank's scatters (into my shard too) and relation gradients are complete
        mark()
        eng.begin_step()
        s0, s1 = eng.slots["ent"]
        if self.lazy:
            _lib.check(eng.lib.kge_optimizer_step_lazy(eng.h, C.byref(eng.opt_cfgs["ent"]), eng.t, p(eng.ent), p(eng.g_ent), p(s0), p(s1),
                                                       self.rps, p(self._stamps), eng.lib.kge_step_stamp(int(step)),
                                                       C.c_void_p(eng.loss_acc.data_ptr() + 8), st))
        else:
            _lib.check(eng.lib.kge_optimizer_step(eng.h, C.byref(eng.opt_cfgs["ent"]), eng.t, p(eng.ent), p(eng.g_ent), p(s0), p(s1),
                                                  self.rps, C.c_void_p(eng.loss_acc.data_ptr() + 8), st))
        lo, hi = self.rel_shard
        r0, r1 = eng.slots["rel"]
        _lib.check(eng.lib.kge_optimizer_step_sharded(
            eng.h, C.byref(eng.opt_cfgs["rel"]), eng.t, self.world, self.rank, self._rel_ptrs, self._grel_ptrs, p(r0), p(r1),
            lo, hi, C.c_void_p(eng.loss_acc.data_ptr() + 8), st))
        mark()
        self.barrier(1)  # all shards updated, relation rows delivered, my relation gradients consumed
        eng.g_rel.zero_()
        mark()
        eng.launches += 6

    def rank_counts(self, triples, side, strategy="worst", filt_off=None, filt_idx=None):
        """full-table rank counts: each rank counts against its shard; the RAW counters {greater, equal, filtered} are
        summed over ranks and the tie strategy is applied once ('middle' = greater + ceil(equal/2) is not additive over
        shards, AbstractScoringLayer.py:232-244)."""
        C, _lib, eng = self._C, self._lib, self.eng
        b = triples.shape[0]
        counts = torch.zeros((b, 3), dtype=torch.int32, device=eng.device)
        p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)
        n_filt = int(filt_idx.numel()) if filt_idx is not None else 0
        ws, ws_bytes = eng.rank_workspace(b, self.rps)
        _lib.check(eng.lib.kge_rank_sharded(eng.h, C.byref(self.map), self.rank, _lib.SIDES[side], _lib.STRATEGIES[strategy],
                                            p(eng.rel), p(triples), b, p(filt_off), p(filt_idx), n_filt, None, p(counts),
                                            p(ws), ws_bytes, eng._stream()))
        allreduce_sum_([counts], self.group)
        return eng.finalize_ranks(counts, strategy)

    def close(self):
        self.eng.close()
