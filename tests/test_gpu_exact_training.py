"""Every training path against the float64 oracle (tests/exact_oracle.py) with NO tolerance.

On tables of coarse dyadic entries every fp32 operation of a training step is exact in any order, so where dL/dscore is
dyadic too (pairwise and absolute_margin with reduction sum, or mean with eta a power of two; KGE_STEP_BACKWARD_EXT with
a dyadic dL/dscore) the kernel's scores, loss and gradient tables must EQUAL the oracle's, element for element: a
dropped, doubled, sign-flipped or misrouted term fails the test however cold its row.  Each test also asserts that the
path it means to exercise ran (residency, bucket entries, deferral, row stash).

The second half runs the losses at their edges (clip bounds of nll / multiclass_nll, hinge ties, saturated
self-adversarial softmax, zero residuals of TransE and RotatE): scores stay exact, gradients are held to a per-element
bound (exact_oracle.within_bound), and a row fed only by clipped scores must be exactly 0."""
import zlib

import numpy as np
import pytest
import torch

import exact_oracle as xo
from ampligraph_b200 import _lib

pytestmark = pytest.mark.gpu

DYADIC_KINDS = ["pairwise", "pairwise_mean", "absolute_margin", "ext"]


def _seed(*a):
    return zlib.crc32(repr(a).encode())


def _engine(*a, **kw):
    from ampligraph_b200.engine import KGEEngine
    return KGEEngine(*a, **kw)


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a)).cuda().contiguous()


def _bucketed_entries(eng):
    """Entries the bucket pre-pass placed in the last step (offset[n_ent] of the workspace's CSR)."""
    ws = eng._train_ws.view(torch.int32)
    off0 = (4 * eng.n_ent + 15) // 16 * 4
    return int(ws[off0 + eng.n_ent].item())


def _loss_setup(kind, eta):
    """(engine loss, loss_params) of a dyadic kind; 'ext' trains with a caller-given dL/dscore."""
    if kind == "pairwise":
        return "pairwise", {"margin": 1.0, "reduction": "sum"}
    if kind == "pairwise_mean":
        assert eta & (eta - 1) == 0, "mean is dyadic only for eta a power of two"
        return "pairwise", {"margin": 0.5, "reduction": "mean"}
    if kind == "absolute_margin":
        return "absolute_margin", {"margin": 1.0, "reduction": "sum"}
    assert kind == "ext"
    return "pairwise", {}


def _negatives(E, t, eta, rng, self_frac=0.05):
    """Uniform injected corruptions; a few replace an entity with itself (N = P exactly)."""
    B = t.shape[0]
    ne = rng.integers(0, E, B * eta).astype(np.int32)
    nk = rng.integers(0, 2, B * eta).astype(np.uint8)
    tiled = np.tile(t, (eta, 1))
    same = rng.random(B * eta) < self_frac
    ne[same] = np.where(nk[same] == 1, tiled[same, 2], tiled[same, 0])
    return ne, nk


def train_exact(model, k, eta, E, R, B, kind, rng, neg_group=0, negatives="injected", triples=None, tables=None,
                setup=None, oracle_device="cpu", chunk=None):
    """One forward_backward on dyadic tables, compared with the float64 oracle for equality.  setup(eng, t) runs after
    the engine is made (hot entities, row stash) and may assert its geometry.  Returns the engine's facts after the step
    (for the caller's path assertions) and the oracle's step."""
    K = xo.internal_k(model, k)
    ent, rel = tables if tables is not None else (xo.grid_table(rng, E, K), xo.grid_table(rng, R, K))
    t = triples if triples is not None else xo.zipf_triples(E, R, B, rng)
    loss, lp = _loss_setup(kind, eta)
    eng = _engine(model, k, eta, E, R, loss=loss, loss_params=lp, neg_group=neg_group)
    if setup is not None:
        setup(eng, t)
    eng.set_embeddings(ent, rel)
    sp = torch.full((B,), float("nan"), device="cuda")
    sn = torch.full((eta * B,), float("nan"), device="cuda")
    if negatives == "philox":
        seed, step = 11, 3
        corr = eng.generate_corruptions(_dev(t), seed=seed, step=step).cpu().numpy()
        neg, ne, nk = None, corr, None
    else:
        ne, nk = negatives if isinstance(negatives, tuple) else _negatives(E, t, eta, rng)
        seed, step, neg = 0, 0, (_dev(ne), _dev(nk))
    ext = {}
    if kind == "ext":
        vals = np.array([-1.0, -0.5, 0.0, 0.5, 1.0], np.float32)
        ext = dict(dpos=rng.choice(vals, B).astype(np.float32), dneg=rng.choice(vals, eta * B).astype(np.float32))
        eng.forward_backward(_dev(t), neg, seed=seed, step=step, mode=_lib.STEP_BACKWARD_EXT,
                             dpos=_dev(ext["dpos"]), dneg=_dev(ext["dneg"]))
    else:
        eng.forward_backward(_dev(t), neg, seed=seed, step=step, scores_pos=sp, scores_neg=sn)
    torch.cuda.synchronize()
    g_ent, ent_pads = xo.dense(eng, eng.g_ent)
    g_rel, rel_pads = xo.dense(eng, eng.g_rel)
    facts = dict(resident=eng.lib.kge_rows_resident(eng.h), loss=eng.read_loss(),
                 bucketed=_bucketed_entries(eng) if getattr(eng, "_train_ws", None) is not None else 0,
                 ws_bytes=int(eng.lib.kge_train_workspace_bytes(eng.h, B)), launches=eng.launches,
                 stash=getattr(eng, "row_stash", None) is not None, hot=list(getattr(eng, "hot_entities", [])))
    eng.close()
    ref = xo.oracle_step(model, ent, rel, t, eta, ne, nk, loss=loss, loss_params=lp, device=oracle_device, chunk=chunk,
                         **ext)
    where = "%s k=%d eta=%d %s" % (model, k, eta, kind)
    for name, x in (("g_ent", ref.g_ent), ("g_rel", ref.g_rel), ("sp", ref.sp), ("sn", ref.sn)):
        xo.assert_fp32_exact(x, where + " oracle " + name)  # the premise: the step is exact in fp32
    if kind != "ext":
        assert torch.equal(sp.cpu().double(), ref.sp.cpu()), where + ": positive scores"
        assert torch.equal(sn.cpu().double(), ref.sn.cpu()), where + ": corruption scores"
        assert facts["loss"] == ref.loss, (where, facts["loss"], ref.loss)
    for name, got, want in (("g_ent", g_ent, ref.g_ent), ("g_rel", g_rel, ref.g_rel)):
        want = want.cpu()
        bad = got != want
        assert not bool(bad.any()), "%s: %s differs in %d elements of %d rows, e.g. row %d: %r vs %r" % (
            where, name, int(bad.sum()), int(bad.any(1).sum()), int(bad.any(1).nonzero()[0]),
            got[bad][:3].tolist(), want[bad][:3].tolist())
    assert ent_pads and rel_pads, where + ": gradient pad columns written"
    return facts, ref


def _force(monkeypatch, kernel=None, sched=None, repl=None, nbuf=None):
    for var, val in (("KGE_B200_TRAIN_KERNEL", kernel), ("KGE_B200_TRAIN_SCHED", sched), ("KGE_B200_TRAIN_REPL", repl),
                     ("KGE_B200_TRAIN_NBUF", nbuf)):
        if val is None:
            monkeypatch.delenv(var, raising=False)
        else:
            monkeypatch.setenv(var, val)


# ---------------------------------------------------------------------------
# the general kernel and the resident fast path (scatter, hot entities, dynamic / static assignment)
# ---------------------------------------------------------------------------
MODEL_K = [("DistMult", 16), ("DistMult", 400), ("ComplEx", 16), ("ComplEx", 200), ("HolE", 8), ("HolE", 128),
           ("TransE", 16), ("TransE", 200)]
PATHS = ["general", "resident", "hot", "dynamic", "static"]
CASES = [pytest.param(m, k, p, kind, id="%s-%d-%s-%s" % (m, k, p, kind))
         for m, k in MODEL_K for p in PATHS for kind in DYADIC_KINDS if m != "TransE" or p == "general"]


@pytest.mark.parametrize("model,k,path,kind", CASES)
def test_exact_general_and_resident_paths(model, k, path, kind, monkeypatch):
    """The resident path runs with the atomic scatter of the replaced rows (KGE_B200_TRAIN_REPL=scatter): the bucketed
    sum has its own tests below.  'hot': kge_set_hot_entities on the static stride; absolute_margin draws Philox
    corruptions, the other kinds inject them."""
    rng = np.random.default_rng(_seed(model, k, path, kind))
    E, R, B, eta = 400, 7, 600, 8
    _force(monkeypatch, kernel="general" if path == "general" else None,
           sched={"dynamic": "dynamic", "static": "static", "hot": "static"}.get(path),
           repl=None if path == "general" else "scatter")

    def setup(eng, t):
        if path == "general":
            assert int(eng.lib.kge_train_workspace_bytes(eng.h, B)) == 0  # nothing buckets under the general kernel
        if path == "hot":
            eng.set_hot_entities(triples=t)
            assert len(eng.hot_entities) == 2

    if path != "general":  # the same engine without the scatter override takes the resident fast path's bucketed step
        monkeypatch.delenv("KGE_B200_TRAIN_REPL")
        probe = _engine(model, k, eta, E, R)
        assert int(probe.lib.kge_train_workspace_bytes(probe.h, B)) > 0, "not the resident fast path"
        probe.close()
        monkeypatch.setenv("KGE_B200_TRAIN_REPL", "scatter")
    facts, _ = train_exact(model, k, eta, E, R, B, kind, rng, setup=setup,
                           negatives="philox" if kind == "absolute_margin" else "injected")
    assert facts["bucketed"] == 0 and facts["ws_bytes"] == 0


# ---------------------------------------------------------------------------
# negative groups, single-buffered groups, column windows, the row stash (all on the general kernel)
# ---------------------------------------------------------------------------
GROUP_CASES = [("DistMult", 16, 3, "2"), ("ComplEx", 16, 3, "2"), ("HolE", 16, 3, "2"), ("TransE", 16, 3, "2"),
               ("DistMult", 16, 3, "1"), ("ComplEx", 200, 3, "1"), ("HolE", 16, 3, "1"), ("TransE", 200, 3, "1"),
               # column windows: half-rows wider than 512 floats
               ("DistMult", 1100, 0, "2"), ("DistMult", 1100, 3, "2"), ("ComplEx", 520, 0, "2"), ("ComplEx", 520, 3, "1"),
               ("HolE", 1024, 0, "2"), ("TransE", 600, 3, "2")]


@pytest.mark.parametrize("model,k,group,nbuf", GROUP_CASES)
@pytest.mark.parametrize("kind", ["pairwise", "ext"])
def test_exact_groups_and_column_windows(model, k, group, nbuf, kind, monkeypatch):
    rng = np.random.default_rng(_seed(model, k, group, nbuf, kind))
    _force(monkeypatch, nbuf=nbuf)
    E, R, B, eta = 300, 5, 200, 7
    facts, _ = train_exact(model, k, eta, E, R, B, kind, rng, neg_group=group)
    assert facts["resident"] == 0 and facts["bucketed"] == 0  # grouped / windowed general kernel, no bucket


@pytest.mark.parametrize("model,k,group", [("ComplEx", 16, 3), ("ComplEx", 520, 0), ("DistMult", 1100, 1), ("TransE", 600, 3),
                                           ("HolE", 16, 3)])
@pytest.mark.parametrize("kind", ["pairwise", "ext"])
def test_exact_row_stash(model, k, group, kind, monkeypatch):
    """kge_set_row_stash: the gradient pass re-reads the replaced rows from the stash (general kernel)."""
    rng = np.random.default_rng(_seed(model, k, group, kind))
    _force(monkeypatch)
    E, R, B, eta = 300, 5, 150, 7

    def setup(eng, t):
        st = eng.ensure_row_stash(B)
        assert st is not None, "expected a geometry that stashes"
        st.fill_(float("nan"))

    facts, _ = train_exact(model, k, eta, E, R, B, kind, rng, neg_group=group, setup=setup)
    assert facts["stash"] and facts["bucketed"] == 0


# ---------------------------------------------------------------------------
# the bucketed replaced-row sum
# ---------------------------------------------------------------------------
BUCKET_SHAPES = [
    ("ComplEx", 16, 8, 700, 600, "injected"), ("HolE", 8, 8, 500, 900, "philox"), ("HolE", 128, 4, 400, 700, "injected"),
    ("DistMult", 400, 20, 3000, 2000, "philox"),  # NIT = 4 rows (cfg3's shape)
    ("ComplEx", 200, 10, 700, 4000, "skewed"), ("DistMult", 33, 5, 700, 4000, "skewed"),  # buckets of thousands
    ("DistMult", 8, 5, 100000, 20000, "philox")]  # 13 tiles of the two-level scan
BUCKET_CASES = [pytest.param(*shape, kind, id="%s-%d-%d-%s-%s" % (shape[0], shape[1], shape[2], shape[5], kind))
                for shape in BUCKET_SHAPES
                for kind in ["pairwise", "absolute_margin", "ext"] + (["pairwise_mean"] if shape[2] & (shape[2] - 1) == 0 else [])]


@pytest.mark.parametrize("model,k,eta,E,B,negs,kind", BUCKET_CASES)
def test_exact_bucketed_sum(model, k, eta, E, B, negs, kind, monkeypatch):
    _force(monkeypatch, repl="gather")
    rng = np.random.default_rng(_seed(model, k, eta, negs, kind))
    R = 9
    t = xo.zipf_triples(E, R, B, rng)
    negatives = negs
    if negs == "skewed":
        negatives = (rng.choice(np.array([3, 77, 500], np.int32), B * eta), rng.integers(0, 2, B * eta).astype(np.uint8))
    facts, _ = train_exact(model, k, eta, E, R, B, kind, rng, triples=t, negatives=negatives)
    assert facts["bucketed"] == eta * B  # the bucketed path ran


def test_exact_cfg2_full_shape(monkeypatch):
    """bench.py's workload shape (ComplEx k=200, eta=10, 14,505 entities, 237 relations, 27,212 Zipf positives) on the
    {-1, -1/2, 0, 1/2, 1} grid with pairwise: ties margin - P + N = 0 are common, so the tie rule is exercised hundreds
    of times.  The oracle runs in float64 on the GPU."""
    _force(monkeypatch)
    rng = np.random.default_rng(2)
    E, R, B, eta = 14505, 237, 27212, 10
    facts, ref = train_exact("ComplEx", 200, eta, E, R, B, "pairwise", rng, oracle_device="cuda", chunk=4096)
    assert facts["bucketed"] == eta * B
    ties = int((1.0 - ref.sp.repeat(eta) + ref.sn == 0).sum())
    assert ties >= 500, ties


# ---------------------------------------------------------------------------
# the deferred step (replaced-row sum + dense optimizer in one owner-per-row launch, two parameter blocks)
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("momentum", [0.0, 0.5])
@pytest.mark.parametrize("reg", [None, {"p": 2, "lambda": 2.0 ** -10}])
@pytest.mark.parametrize("model,k", [("ComplEx", 16), ("DistMult", 33), ("HolE", 8)])
def test_exact_deferred_sgd(model, k, momentum, reg, monkeypatch):
    """SGD at lr = 2^-6 on dyadic gradients is exact, so the tables after each deferred step equal the oracle's bit
    for bit.  Before the second step the tables are reset to a fresh dyadic grid (the first step's update leaves it);
    the momentum slot carries over.  The two steps write the two parameter blocks in turn."""
    _force(monkeypatch)
    rng = np.random.default_rng(_seed(model, k, momentum, str(reg)))
    E, R, B, eta, lr = 500, 9, 1000, 4, 2.0 ** -6
    K = xo.internal_k(model, k)
    lp = {"margin": 1.0}
    params = {"learning_rate": lr, "momentum": momentum}
    eng = _engine(model, k, eta, E, R, loss="pairwise", loss_params=lp, optimizer="sgd", optimizer_params=params,
                  regularizer=reg)
    lam = reg["lambda"] if reg else 0.0
    acc = [None, None]
    blocks = []
    for step in range(2):
        ent, rel = xo.grid_table(rng, E, K), xo.grid_table(rng, R, K)
        eng.set_embeddings(ent, rel)
        t = xo.zipf_triples(E, R, B, rng)
        if step == 0:
            ne, nk = _negatives(E, t, eta, rng)
            neg, seed = (_dev(ne), _dev(nk)), 0
        else:
            seed = 5
            ne, nk, neg = eng.generate_corruptions(_dev(t), seed=seed, step=step).cpu().numpy(), None, None
        launches = eng.launches
        eng.forward_backward(_dev(t), neg, seed=seed, step=step, defer=True)
        assert eng._deferred
        eng.apply_gradients()
        assert not eng._deferred and eng.launches - launches == 5  # pre-pass (3), fused kernel, deferred sum + optimizer
        blocks.append(eng._pblock.data_ptr())
        ref = xo.oracle_step(model, ent, rel, t, eta, ne, nk, loss="pairwise", loss_params=lp)
        new = []
        for i, (x0, g) in enumerate(((ent, ref.g_ent), (rel, ref.g_rel))):
            x0 = torch.as_tensor(x0, dtype=torch.float64)
            gg = g + 2.0 * lam * x0  # the L2 term's gradient at the pre-update value
            if momentum == 0.0:
                new.append(x0 - lr * gg)
            else:
                acc[i] = (momentum * acc[i] if acc[i] is not None else 0.0) - lr * gg
                new.append(x0 + acc[i])
            xo.assert_fp32_exact(new[-1], "updated table")
        got_e, pe = xo.dense(eng, eng.ent)
        got_r, pr = xo.dense(eng, eng.rel)
        assert torch.equal(got_e, new[0]) and torch.equal(got_r, new[1]), (step, (got_e - new[0]).abs().max())
        assert pe and pr  # pads of the block the step wrote
        reg_loss = lam * (float((torch.as_tensor(ent, dtype=torch.float64) ** 2).sum())
                          + float((torch.as_tensor(rel, dtype=torch.float64) ** 2).sum()))
        assert eng.read_loss() == ref.loss + reg_loss
    assert blocks[0] != blocks[1]  # each step wrote the other parameter block
    eng.close()


# ---------------------------------------------------------------------------
# the losses' edges
# ---------------------------------------------------------------------------
def _run_rows(model, k, eta, ent, rel, t, ne, nk, loss, lp, kernel=None, monkeypatch=None, neg_group=0):
    """forward_backward on explicit tables / corruptions -> (scores pos, scores neg, g_ent, g_rel, loss) on the host."""
    _force(monkeypatch, kernel=kernel)
    E, R, B = ent.shape[0], rel.shape[0], t.shape[0]
    eng = _engine(model, k, eta, E, R, loss=loss, loss_params=lp, neg_group=neg_group)
    eng.set_embeddings(ent, rel)
    sp, sn = torch.empty(B, device="cuda"), torch.empty(eta * B, device="cuda")
    eng.forward_backward(_dev(t), (_dev(ne), _dev(nk)), scores_pos=sp, scores_neg=sn)
    torch.cuda.synchronize()
    out = (sp.cpu().double(), sn.cpu().double(), xo.dense(eng, eng.g_ent)[0], xo.dense(eng, eng.g_rel)[0], eng.read_loss())
    eng.close()
    return out


def _check_bound(model, ent, rel, t, ref, got_e, got_r, extra, where):
    (Ae, A1e, ne_), (Ar, A1r, nr_) = xo.grad_bound(model, ent, rel, t, ref.corr, ref.mag_pos, ref.mag_neg)
    for name, got, want, A, A1, n in (("g_ent", got_e, ref.g_ent, Ae, A1e, ne_), ("g_rel", got_r, ref.g_rel, Ar, A1r, nr_)):
        assert bool(torch.isfinite(got).all()), (where, name)
        ok, ratio = xo.within_bound(got, want, A, A1, n, extra)
        assert ok, (where, name, ratio)
    return Ae


CLIP_TARGETS = [-75.0 - 2.0 ** -4, -75.0, 75.0, 75.0 + 2.0 ** -4, 200.0, -200.0]


def _clip_rows(eta):
    """DistMult k = 8, relation row and object row of ones: a subject's score is the sum of its row.  Positive b has
    subject S_b with score CLIP_TARGETS[b]; its corruption 0 replaces the subject by X_b (same score), the others by
    the zero row Y.  S_b and X_b appear nowhere else: each is fed by one edge score only.
    Entities: 0 = object, 1 = Y, 2 + b = S_b, 8 + b = X_b."""
    n = len(CLIP_TARGETS)
    ent = np.zeros((2 + 2 * n, 8), np.float32)
    ent[0] = 1.0
    for b, target in enumerate(CLIP_TARGETS):
        ent[2 + b] = ent[2 + n + b] = target / 8.0
    rel = np.ones((1, 8), np.float32)
    t = np.array([[2 + b, 0, 0] for b in range(n)], np.int32)
    ne = np.ones((eta, n), np.int32)
    ne[0] = 2 + n + np.arange(n)
    nk = np.zeros((eta, n), np.uint8)  # every corruption replaces the subject
    return ent, rel, t, ne.reshape(-1), nk.reshape(-1)


LOSS_EXTRA = {"nll": 16, "multiclass_nll": None, "self_adversarial": None}  # None: 2 eta + 16 (sums over eta terms)


def _extra(loss, eta):
    e = LOSS_EXTRA[loss]
    return 2 * eta + 16 if e is None else e


@pytest.mark.parametrize("loss", ["nll", "multiclass_nll"])
@pytest.mark.parametrize("reduction", ["sum", "mean"])
@pytest.mark.parametrize("kernel", [None, "general"])
def test_edge_clip_bounds(loss, reduction, kernel, monkeypatch):
    """Scores at -75 - 2^-4, -75, 75, 75 + 2^-4, 200 and -200: the clip masks inP / inN pass the gradient at exactly
    +-75 and nowhere beyond.  A row fed only by a clipped score is exactly 0; one fed by a boundary score is not."""
    eta = 8
    ent, rel, t, ne, nk = _clip_rows(eta)
    lp = {"reduction": reduction}
    sp, sn, g_e, g_r, _ = _run_rows("DistMult", 8, eta, ent, rel, t, ne, nk, loss, lp, kernel, monkeypatch)
    ref = xo.oracle_step("DistMult", ent, rel, t, eta, ne, nk, loss=loss, loss_params=lp)
    targets = torch.tensor(CLIP_TARGETS, dtype=torch.float64)
    assert torch.equal(ref.sp, targets) and torch.equal(ref.sn.reshape(eta, -1)[0], targets)
    assert torch.equal(sp, ref.sp) and torch.equal(sn, ref.sn)
    A = _check_bound("DistMult", ent, rel, t, ref, g_e, g_r, _extra(loss, eta), (loss, reduction, kernel))
    n = len(CLIP_TARGETS)
    for b, target in enumerate(CLIP_TARGETS):
        for row in (2 + b, 2 + n + b):
            if abs(target) > 75.0:
                assert bool((ref.g_ent[row] == 0).all()) and bool((g_e[row] == 0).all()), (loss, target, row)
            else:
                assert bool((ref.g_ent[row] != 0).all()), (loss, target, row)
                # nonzero wherever the oracle's value exceeds what fp32 can lose on the way
                if bool((ref.g_ent[row].abs() > (1 + 8 + _extra(loss, eta)) * xo.FP32_EPS * A[row]).all()):
                    assert bool((g_e[row] != 0).all()), (loss, target, row)
    # every boundary row survives in fp32 here: S_-75, S_75, X_-75, X_75 (the construction keeps each D moderate)
    must = [2 + 1, 2 + 2, 2 + n + 1, 2 + n + 2]
    assert all(bool((g_e[r] != 0).all()) for r in must), [(r, g_e[r, 0].item()) for r in must]


@pytest.mark.parametrize("loss,margin", [("pairwise", 1.0), ("absolute_margin", 1.0)])
@pytest.mark.parametrize("kernel", [None, "general"])
def test_edge_hinge_ties(loss, margin, kernel, monkeypatch):
    """margin - P + N (pairwise) or margin + N (absolute_margin) at exactly 0 and one grid step (2^-4) on either side:
    TF's maximum() gives the tie to its first argument, so the tied corruption's row receives the gradient."""
    eta = 4
    P = 0.5
    base = -(margin - P) if loss == "pairwise" else -margin  # the tied corruption score
    negs = [base - 2.0 ** -4, base, base + 2.0 ** -4]
    ent = np.zeros((2 + 2 + 3, 8), np.float32)  # 0 object, 1 Y (zero row), 2 S (positive), 3 unused, 4.. X_j
    ent[0] = 1.0
    ent[2] = P / 8.0
    for j, v in enumerate(negs):
        ent[4 + j] = v / 8.0
    rel = np.ones((1, 8), np.float32)
    t = np.array([[2, 0, 0]] * 3, np.int32)  # three positives, one edge corruption each
    ne = np.ones((eta, 3), np.int32)
    ne[0] = [4, 5, 6]
    nk = np.zeros((eta, 3), np.uint8)
    ne, nk = ne.reshape(-1), nk.reshape(-1)
    lp = {"margin": margin, "reduction": "sum"}
    sp, sn, g_e, g_r, got_loss = _run_rows("DistMult", 8, eta, ent, rel, t, ne, nk, loss, lp, kernel, monkeypatch)
    ref = xo.oracle_step("DistMult", ent, rel, t, eta, ne, nk, loss=loss, loss_params=lp)
    assert torch.equal(ref.sn.reshape(eta, -1)[0], torch.tensor(negs, dtype=torch.float64))
    assert torch.equal(sp, ref.sp) and torch.equal(sn, ref.sn) and got_loss == ref.loss
    assert torch.equal(g_e, ref.g_ent) and torch.equal(g_r, ref.g_rel)
    assert bool((g_e[4] == 0).all()) and bool((g_e[5] != 0).all()) and bool((g_e[6] != 0).all())


@pytest.mark.parametrize("eta", [7, 32, 33, 70])
@pytest.mark.parametrize("kernel", [None, "general"])
def test_edge_self_adversarial_saturated(eta, kernel, monkeypatch):
    """eta <= 32 (one corruption per lane) and eta > 32 (the looped code path): positive 0's corruption scores are 97 and
    -103 (N + margin = +-100; alpha N spread 100, so every softmax weight but one underflows); positive 1's are spread
    over a few units (no saturation); positive 2's corruption 0 replaces the subject with itself (N = P)."""
    m, alpha = 3.0, 0.5
    B = 3
    E = 3 + B * eta
    ent = np.zeros((E, 8), np.float32)
    ent[0] = 1.0                      # object
    ent[1], ent[2] = 0.5 / 8, -1.0 / 8  # subjects: P = 0.5, -1
    t = np.array([[1, 0, 0], [2, 0, 0], [1, 0, 0]], np.int32)
    ne = np.zeros((eta, B), np.int32)
    for b in range(B):
        for j in range(eta):
            x = 3 + b * eta + j
            ne[j, b] = x
            if b == 0:
                ent[x] = (97.0 if j == 0 else -103.0) / 8
            elif b == 1:
                ent[x] = (j % 9 - 4) * 0.25 / 8
            else:
                ent[x] = ((j % 5) - 2) * 0.5 / 8
    ne[0, 2] = 1  # N = P
    nk = np.zeros((eta, B), np.uint8)
    ne, nk = ne.reshape(-1), nk.reshape(-1)
    rel = np.ones((1, 8), np.float32)
    lp = {"margin": m, "alpha": alpha, "reduction": "sum"}
    sp, sn, g_e, g_r, got_loss = _run_rows("DistMult", 8, eta, ent, rel, t, ne, nk, "self_adversarial", lp, kernel,
                                           monkeypatch)
    ref = xo.oracle_step("DistMult", ent, rel, t, eta, ne, nk, loss="self_adversarial", loss_params=lp)
    assert float(ref.sn[0]) + m == 100.0 and float(ref.sn[B]) + m == -100.0
    assert float(ref.sn[2]) == float(ref.sp[2])
    assert torch.equal(sp, ref.sp) and torch.equal(sn, ref.sn)
    _check_bound("DistMult", ent, rel, t, ref, g_e, g_r, _extra("self_adversarial", eta), (eta, kernel))
    assert abs(got_loss - ref.loss) <= 1e-6 * abs(ref.loss)


@pytest.mark.parametrize("group", [0, 3])
def test_edge_transe_zero_residual(group, monkeypatch):
    """TransE columns whose residual is exactly 0, on the positive, on an object-replaced corruption (s + p - r = 0) and
    on a subject-replaced one (r + p - o = 0): |x|'(0) = 0, so those columns of the rows involved get exactly 0; the
    other columns do not."""
    rng = np.random.default_rng(3)
    k, eta = 8, 4
    E = 12
    ent = xo.grid_table(rng, E, k)
    rel = xo.grid_table(rng, 2, k)
    S, O, Xo, Xs = 0, 1, 2, 3
    ent[O, :4] = ent[S, :4] + rel[0, :4]   # positive: zero residual in columns 0..3
    ent[O, 4:] = ent[S, 4:] + rel[0, 4:] - 0.5  # and residual +1/2 elsewhere
    ent[Xo] = ent[S] + rel[0]              # object replaced: s + p - Xo = 0 in columns 0..3, +1 elsewhere
    ent[Xo, 4:] -= 1.0
    ent[Xs] = ent[O] - rel[0]              # subject replaced: Xs + p - o = 0 in columns 0..3, -1 elsewhere
    ent[Xs, 4:] -= 1.0
    t = np.array([[S, 0, O]], np.int32)
    ne = np.array([Xo, Xs, Xo, Xs], np.int32)
    nk = np.array([1, 0, 1, 0], np.uint8)
    lp = {"margin": 16.0, "reduction": "sum"}  # every hinge active
    sp, sn, g_e, g_r, got_loss = _run_rows("TransE", k, eta, ent, rel, t, ne, nk, "pairwise", lp, None, monkeypatch,
                                           neg_group=group)
    ref = xo.oracle_step("TransE", ent, rel, t, eta, ne, nk, loss="pairwise", loss_params=lp)
    assert torch.equal(sp, ref.sp) and torch.equal(sn, ref.sn) and got_loss == ref.loss
    assert torch.equal(g_e, ref.g_ent) and torch.equal(g_r, ref.g_rel)
    for row in (S, O, Xo, Xs):
        assert bool((g_e[row, :4] == 0).all()) and bool((g_e[row, 4:] != 0).all()), row
    assert bool((g_r[0, :4] == 0).all()) and bool((g_r[0, 4:] != 0).all())


@pytest.mark.parametrize("kernel", [None, "general"])
def test_edge_rotate_zero_modulus(kernel, monkeypatch):
    """RotatE with a theta = 0 relation row and s = o: the residual R(0) s - o is exactly 0, where the reference's sqrt
    gradient is NaN and the kernel's rot_unit returns 0.  Positive 0 is (A, 0, A'), A' a copy of A, and its corruptions
    replace the subject by A itself or the object by A'': every one of its residuals is 0, so A, A', A'' get exactly 0.
    Positive 1 is (C, 0, C') with C' = C in the first k/2 complex columns only: those columns of C, C' and of the
    relation row's angle get exactly 0, the others do not.  The gradient is finite everywhere."""
    rng = np.random.default_rng(5)
    k, eta, E, R = 8, 4, 40, 3
    ent = xo.dyadic_table(rng, E, 2 * k, frac_bits=2)
    rel = xo.dyadic_table(rng, R, 2 * k, frac_bits=2)
    rel[0] = 0.0
    A, A1, A2, C, C1 = 0, 1, 2, 3, 4
    ent[A1] = ent[A2] = ent[A]
    h = k // 2
    ent[C] = 0.5  # y = R(0) C = C: the angle's gradient a y_im - b y_re is nonzero where the residual is
    ent[C1] = ent[C]
    ent[C1, h:k] += 0.5
    ent[C1, k + h:] -= 0.25
    t = np.array([[A, 0, A1], [C, 0, C1]] + [[10 + i, 1 + i % 2, 20 + i] for i in range(6)], np.int32)
    B = t.shape[0]
    ne = rng.integers(5, E, (eta, B)).astype(np.int32)
    nk = rng.integers(0, 2, (eta, B)).astype(np.uint8)
    ne[:, 0] = [A, A2, A, A2]
    nk[:, 0] = [0, 1, 0, 1]
    ne[:, 1] = C1
    nk[:, 1] = 1  # object replaced by C' itself
    ne, nk = ne.reshape(-1), nk.reshape(-1)
    lp = {"margin": 3.0, "alpha": 0.5}
    sp, sn, g_e, g_r, _ = _run_rows("RotatE", k, eta, ent, rel, t, ne, nk, "self_adversarial", lp, kernel, monkeypatch)
    ref = xo.oracle_step("RotatE", ent, rel, t, eta, ne, nk, loss="self_adversarial", loss_params=lp, rot_table=True)
    for x in (g_e, g_r, ref.g_ent, ref.g_rel):
        assert bool(torch.isfinite(x).all())
    assert float(ref.sp[0]) == 0.0 and float(sp[0]) == 0.0
    for row in (A, A1, A2):
        assert bool((g_e[row] == 0).all()) and bool((ref.g_ent[row] == 0).all()), row
    zero_cols = np.r_[0:h, k:k + h]
    for row in (C, C1):
        assert bool((g_e[row, zero_cols] == 0).all()), row
        assert bool((g_e[row, np.r_[h:k, k + h:2 * k]] != 0).all()), row
    assert bool((g_r[0, :h] == 0).all()) and bool((g_r[0, h:k] != 0).all())
    bound = xo.RotatEBound(ent, rel, t, ref, eta, loss="self_adversarial", loss_params=lp)
    for name, ok, ratio in bound.check(g_e, g_r, ref.g_ent, ref.g_rel):
        assert ok, (kernel, name, ratio)
    assert bound.check_scores(sp, ref.sp, "sp")[0] and bound.check_scores(sn, ref.sn, "sn")[0]
