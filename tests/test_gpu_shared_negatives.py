"""Shared negatives (kge_shared_negatives_step, DESIGN.md 3.21) against the float64 oracle (tests/exact_oracle.py), run
on the corruptions tests/shared_negatives_oracle.py materialises.

On coarse dyadic tables with dyadic dL/dscore (pairwise, pairwise mean with eta a power of two, absolute_margin) every
fp32 operation is exact in any order, so the step's loss, g_ent and g_rel must EQUAL the oracle's, element for element,
pad columns 0.  The other losses and RotatE are held to exact_oracle's per-element bounds (TrilinearBound, RotatEBound),
and each bounded case shows the check is sensitive: the kernel's output fails it against an oracle with one
corruption's dL/dscore multiplied by 1 + 2^-10 (RotatE: with one corruption dropped)."""
import zlib

import numpy as np
import pytest
import torch

import exact_oracle as xo
import shared_negatives_oracle as sno
from ampligraph_b200 import _lib
from ampligraph_b200.engine import NegativeSamplerTables, shared_negatives_workspace_bytes

pytestmark = pytest.mark.gpu

SEED, STEP = 5, 3


def _rng(*a):
    return np.random.default_rng(zlib.crc32(repr(a).encode()))


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a)).cuda().contiguous()


def _engine(model, k, eta, E, R, loss, lp, **kw):
    from ampligraph_b200.engine import KGEEngine
    return KGEEngine(model, k, eta, E, R, loss=loss, loss_params=lp, **kw)


def _glorot(rng, rows, K):
    lim = np.sqrt(6.0 / (rows + K))
    return rng.uniform(-lim, lim, (rows, K)).astype(np.float32)


def shared_step(model, k, eta, E, R, C, loss, lp, ent, rel, t, sampler_tables=None, seed=SEED):
    """One kge_shared_negatives_step -> (g_ent, g_rel dense float64, pads all zero, loss)."""
    eng = _engine(model, k, eta, E, R, loss, lp)
    eng.set_embeddings(ent, rel)
    sampler = NegativeSamplerTables(sampler_tables, 1, eng.device) if sampler_tables is not None else None
    n0 = eng.launches
    eng.shared_negatives_backward(_dev(t), C, seed=seed, step=STEP, sampler=sampler)
    torch.cuda.synchronize()
    assert eng.launches - n0 == 3 + (model == "RotatE")
    g_ent, ep = xo.dense(eng, eng.g_ent)
    g_rel, rp = xo.dense(eng, eng.g_rel)
    loss_v = eng.read_loss()
    eng.close()
    return g_ent, g_rel, ep and rp, loss_v


def _kind(kind):
    return {"pairwise": ("pairwise", {"margin": 1.0, "reduction": "sum"}),
            "pairwise_mean": ("pairwise", {"margin": 0.5, "reduction": "mean"}),
            "absolute_margin": ("absolute_margin", {"margin": 1.0, "reduction": "sum"})}[kind]


# (C, eta, B, kind): C in {1, 3, 32, B} with B not a multiple of C, eta in {1, 7, 33, 256}
EXACT = [(1, 7, 13, "pairwise"), (3, 33, 20, "absolute_margin"), (32, 1, 40, "pairwise"), (50, 256, 50, "pairwise_mean"),
         (3, 256, 37, "absolute_margin")]
MODEL_K = [("TransE", 16), ("TransE", 200), ("DistMult", 16), ("DistMult", 400), ("ComplEx", 16), ("ComplEx", 200),
           ("HolE", 16), ("HolE", 128)]


def run_exact(model, k, C, eta, B, kind, E=300, R=7):
    rng = _rng(model, k, C, eta, B, kind, E)
    K = xo.internal_k(model, k)
    ent, rel = xo.grid_table(rng, E, K), xo.grid_table(rng, R, K)
    t = xo.zipf_triples(E, R, B, rng) if E > 2 else np.stack(
        [rng.integers(0, E, B), rng.integers(0, R, B), rng.integers(0, E, B)], 1).astype(np.int32)
    loss, lp = _kind(kind)
    g_ent, g_rel, pads, loss_v = shared_step(model, k, eta, E, R, C, loss, lp, ent, rel, t)
    ne, nk = sno.sample(t, eta, E, SEED, STEP, C)
    ref = xo.oracle_step(model, ent, rel, t, eta, ne, nk, loss=loss, loss_params=lp, device="cuda")
    where = "%s k=%d C=%d eta=%d B=%d %s E=%d" % (model, k, C, eta, B, kind, E)
    for name, x in (("g_ent", ref.g_ent), ("g_rel", ref.g_rel), ("sp", ref.sp), ("sn", ref.sn)):
        xo.assert_fp32_exact(x, where + " oracle " + name)
    assert loss_v == ref.loss, (where, loss_v, ref.loss)
    for name, got, want in (("g_ent", g_ent, ref.g_ent.cpu()), ("g_rel", g_rel, ref.g_rel.cpu())):
        bad = got != want
        assert not bool(bad.any()), "%s: %s differs in %d elements" % (where, name, int(bad.sum()))
    assert pads, where + ": gradient pad columns written"
    return ne, nk, t


@pytest.mark.parametrize("model,k", MODEL_K)
@pytest.mark.parametrize("C,eta,B,kind", EXACT)
def test_exact(model, k, C, eta, B, kind):
    ne, nk, t = run_exact(model, k, C, eta, B, kind)
    if C > 1 and eta > 1:  # the chunk's positives really shared their candidates
        assert (ne.reshape(eta, B)[:, 1] == ne.reshape(eta, B)[:, 0]).all()


@pytest.mark.parametrize("model,k", [("TransE", 16), ("DistMult", 16), ("ComplEx", 16), ("HolE", 16)])
def test_exact_two_entities(model, k):
    """n_ent = 2: duplicate candidates everywhere, and candidates equal to the positives' own entities."""
    ne, nk, t = run_exact(model, k, 4, 33, 21, "absolute_margin", E=2, R=2)
    tiled = np.tile(t, (33, 1))
    assert (ne == np.where(nk == 1, tiled[:, 2], tiled[:, 0])).any()


def test_exact_eta_1024():
    run_exact("DistMult", 16, 16, 1024, 40, "pairwise_mean")


# ---------------------------------------------------------------------------
# bounded cases
# ---------------------------------------------------------------------------
SA = ("self_adversarial", {"margin": 3.0, "alpha": 0.5})
BOUNDED = [("nll", {}), ("multiclass_nll", {}), ("multiclass_nll", {"reduction": "mean"}), SA,
           ("nll", {"reduction": "mean"})]
ROT_LOSSES = BOUNDED + [("pairwise", {"margin": 0.5})]


def run_bounded(model, k, C, eta, B, loss, lp, E=200, R=5):
    rng = _rng(model, k, C, eta, B, loss, repr(lp))
    K = xo.internal_k(model, k)
    ent, rel = _glorot(rng, E, K), _glorot(rng, R, K)
    t = xo.zipf_triples(E, R, B, rng)
    g_ent, g_rel, pads, loss_v = shared_step(model, k, eta, E, R, C, loss, lp, ent, rel, t)
    ne, nk = sno.sample(t, eta, E, SEED, STEP, C)
    kw = dict(rot_table=True) if model == "RotatE" else {}
    ref = xo.oracle_step(model, ent, rel, t, eta, ne, nk, loss=loss, loss_params=lp, device="cuda", **kw)
    if model == "RotatE":
        bound = xo.RotatEBound(ent, rel, t, ref, eta, loss, lp, device="cuda")
    else:
        bound = xo.TrilinearBound(model, ent, rel, t, ref, eta, loss, lp, device="cuda")
    where = "%s k=%d C=%d eta=%d %s %r" % (model, k, C, eta, loss, lp)
    res = bound.check(g_ent, g_rel, ref.g_ent, ref.g_rel)
    print(where, res)
    assert all(ok for _, ok, _ in res), (where, res)
    assert abs(loss_v - ref.loss) <= float(bound.loss_err) + 1e-12, (where, loss_v, ref.loss)
    assert pads
    # sensitivity: one corruption's dL/dscore times 1 + 2^-10 (RotatE: the corruption dropped, as its own tests do)
    factor = -1.0 if model == "RotatE" else 2.0 ** -10
    pert = xo.perturbed_term(model, ent, rel, t, ref, eta, factor, max_lookups=None, device="cuda", **kw)
    assert pert is not None
    _, one = pert
    res = bound.check(g_ent, g_rel, ref.g_ent + one.g_ent, ref.g_rel + one.g_rel)
    assert not all(ok for _, ok, _ in res), where + ": the check is not sensitive to one corruption"


@pytest.mark.parametrize("model,k", [("TransE", 50), ("DistMult", 50), ("ComplEx", 50), ("HolE", 64), ("ComplEx", 1000)])
@pytest.mark.parametrize("loss,lp", BOUNDED)
def test_bounded(model, k, loss, lp):
    run_bounded(model, k, 8, 33, 40, loss, lp)


@pytest.mark.parametrize("k", [50, 1000])
@pytest.mark.parametrize("loss,lp", ROT_LOSSES)
def test_rotate_bounded(k, loss, lp):
    run_bounded("RotatE", k, 8, 33 if k == 50 else 9, 40 if k == 50 else 12, loss, lp)


# ---------------------------------------------------------------------------
# the losses' edges (as test_gpu_exact_training.py's test_edge_*): the chunks' candidates are drawn first
# (shared_negatives_oracle.candidates), then their rows of the table are set to build each edge.  Edge candidates sit
# in the second tile of 32 (j >= 32), whose CTAs add the kept rows' terms with gP = 0.
# ---------------------------------------------------------------------------
EDGE_E = 1 << 14
ALWAYS_SUBJECT = np.array([0xFFFFFFFF] * 3, np.uint32)  # Bernoulli thresholds: the subject is replaced unless x = 2^32 - 1


def _edge_seed(B, C, eta, rels, thr=None, ok=lambda cand, nk: True):
    """The first seed from 100 whose candidates are pairwise distinct and for which ok(cand [n_chunks, eta], nk [eta,
    B]) holds (nk: the sides of positives with relations `rels`) -> (seed, cand, nk, ids outside the candidates)."""
    t = np.zeros((B, 3), np.int32)
    t[:, 1] = rels
    for seed in range(100, 1100):
        cand = sno.candidates(B, C, eta, EDGE_E, seed, STEP)
        if np.unique(cand).size != cand.size:
            continue
        nk = sno.sample(t, eta, EDGE_E, seed, STEP, C, thresholds=thr)[1].reshape(eta, B)
        if ok(cand, nk):
            used = set(cand.ravel().tolist())
            return seed, cand, nk, [e for e in range(EDGE_E) if e not in used]
    raise AssertionError("no seed gives distinct candidates")


def _oracle(model, ent, rel, t, eta, seed, C, loss, lp, thr=None):
    ne, nk = sno.sample(t, eta, EDGE_E, seed, STEP, C, thresholds=thr)
    kw = dict(rot_table=True) if model == "RotatE" else {}
    return xo.oracle_step(model, ent, rel, t, eta, ne, nk, loss=loss, loss_params=lp, **kw)


def _within(model, ent, rel, t, ref, got_e, got_r, extra, where):
    (Ae, A1e, ne_), (Ar, A1r, nr_) = xo.grad_bound(model, ent, rel, t, ref.corr, ref.mag_pos, ref.mag_neg)
    for name, got, want, A, A1, n in (("g_ent", got_e, ref.g_ent, Ae, A1e, ne_), ("g_rel", got_r, ref.g_rel, Ar, A1r, nr_)):
        assert bool(torch.isfinite(got).all()), (where, name)
        ok, ratio = xo.within_bound(got, want, A, A1, n, extra)
        assert ok, (where, name, ratio)
    return Ae


CLIP_TARGETS = [-75.0 - 2.0 ** -4, -75.0, 75.0, 75.0 + 2.0 ** -4, 200.0, -200.0]


@pytest.mark.parametrize("loss", ["nll", "multiclass_nll"])
@pytest.mark.parametrize("reduction", ["sum", "mean"])
def test_edge_clip_bounds(loss, reduction):
    """DistMult k = 8, relation row and object row of ones, every subject replaced: a score is the sum of its subject
    row.  Chunk b (C = 2) holds two positives with subjects S_b, S'_b of score CLIP_TARGETS[b]; its candidate 33 has
    the same score, the others the zero row's 0.  The clip masks pass the gradient at exactly +-75 and nowhere beyond:
    a row fed only by clipped scores is exactly 0, one fed by a boundary score is not."""
    n, eta, C = len(CLIP_TARGETS), 40, 2
    B = C * n
    seed, cand, nk, free = _edge_seed(B, C, eta, 0, ALWAYS_SUBJECT, lambda c, k: bool((k == 0).all()))
    O, S = free[0], np.array(free[1:1 + B]).reshape(n, C)
    ent = np.zeros((EDGE_E, 8), np.float32)
    ent[O] = 1.0
    for b, target in enumerate(CLIP_TARGETS):
        ent[S[b]] = ent[cand[b, 33]] = target / 8.0
    rel = np.ones((3, 8), np.float32)
    t = np.array([[S[b, c], 0, O] for b in range(n) for c in range(C)], np.int32)
    lp = {"reduction": reduction}
    tabs = {"thresholds": ALWAYS_SUBJECT, "pools": None, "filter": None}
    g_e, g_r, pads, _ = shared_step("DistMult", 8, eta, EDGE_E, 3, C, loss, lp, ent, rel, t, tabs, seed=seed)
    ref = _oracle("DistMult", ent, rel, t, eta, seed, C, loss, lp, ALWAYS_SUBJECT)
    targets = torch.tensor(np.repeat(CLIP_TARGETS, C), dtype=torch.float64)
    assert torch.equal(ref.sp, targets) and torch.equal(ref.sn.reshape(eta, -1)[33], targets)
    extra = 16 if loss == "nll" else 2 * eta + 16
    A = _within("DistMult", ent, rel, t, ref, g_e, g_r, extra, (loss, reduction))
    assert pads
    for b, target in enumerate(CLIP_TARGETS):
        for row in (S[b, 0], S[b, 1], cand[b, 33]):
            if abs(target) > 75.0:
                assert bool((ref.g_ent[row] == 0).all()) and bool((g_e[row] == 0).all()), (loss, target, row)
            else:
                assert bool((ref.g_ent[row] != 0).all()), (loss, target, row)
                if bool((ref.g_ent[row].abs() > (1 + 8 + extra) * xo.FP32_EPS * A[row]).all()):
                    assert bool((g_e[row] != 0).all()), (loss, target, row)
    must = [S[1, 0], S[2, 0], cand[1, 33], cand[2, 33]]  # the boundary rows survive in fp32 here
    assert all(bool((g_e[r] != 0).all()) for r in must), [(r, g_e[r, 0].item()) for r in must]


@pytest.mark.parametrize("loss,margin", [("pairwise", 1.0), ("absolute_margin", 1.0)])
def test_edge_hinge_ties(loss, margin):
    """One chunk of three positives of score 1/2 (every subject replaced); candidates 33, 34, 35 put margin - P + N
    (pairwise) or margin + N (absolute_margin) one grid step (2^-4) below 0, at exactly 0 and one step above, the others
    score 0.  TF's maximum() gives the tie to its first argument, so the tied candidate's row receives the gradient and
    the one below does not; loss and gradients equal the oracle's."""
    eta, B, P = 36, 3, 0.5
    base = -(margin - P) if loss == "pairwise" else -margin
    negs = [base - 2.0 ** -4, base, base + 2.0 ** -4]
    seed, cand, nk, free = _edge_seed(B, B, eta, 0, ALWAYS_SUBJECT, lambda c, k: bool((k == 0).all()))
    O, S = free[0], free[1:1 + B]
    ent = np.zeros((EDGE_E, 8), np.float32)
    ent[O] = 1.0
    ent[S] = P / 8.0
    for j, v in zip((33, 34, 35), negs):
        ent[cand[0, j]] = v / 8.0
    rel = np.ones((3, 8), np.float32)
    t = np.array([[x, 0, O] for x in S], np.int32)
    lp = {"margin": margin, "reduction": "sum"}
    tabs = {"thresholds": ALWAYS_SUBJECT, "pools": None, "filter": None}
    g_e, g_r, pads, got_loss = shared_step("DistMult", 8, eta, EDGE_E, 3, B, loss, lp, ent, rel, t, tabs, seed=seed)
    ref = _oracle("DistMult", ent, rel, t, eta, seed, B, loss, lp, ALWAYS_SUBJECT)
    assert torch.equal(ref.sn.reshape(eta, -1)[33:36, 0], torch.tensor(negs, dtype=torch.float64))
    assert got_loss == ref.loss
    assert torch.equal(g_e, ref.g_ent) and torch.equal(g_r, ref.g_rel) and pads
    lo, tie, hi = cand[0, 33], cand[0, 34], cand[0, 35]
    assert bool((g_e[lo] == 0).all()) and bool((g_e[tie] != 0).all()) and bool((g_e[hi] != 0).all())


def test_edge_transe_zero_residual():
    """TransE columns whose residual is exactly 0 on the positive (s + p - o), on every object-replaced corruption
    (s + p - c) and on every subject-replaced one (c + p - o): |x|'(0) = 0, so those columns of every row involved get
    exactly 0 and the other columns do not.  One positive, 36 candidates over two tiles, both sides drawn."""
    k, eta = 8, 36
    seed, cand, nk, free = _edge_seed(1, 1, eta, 0, None, lambda c, s: 0 < int(s.sum()) < eta)
    rng = np.random.default_rng(3)
    ent = xo.grid_table(rng, EDGE_E, k)
    rel = xo.grid_table(rng, 2, k)
    S, O = free[0], free[1]
    ent[O, :4] = ent[S, :4] + rel[0, :4]        # positive: zero residual in columns 0..3
    ent[O, 4:] = ent[S, 4:] + rel[0, 4:] - 0.5  # and residual +1/2 elsewhere
    for j in range(eta):
        c = cand[0, j]
        if nk[j, 0]:  # object replaced: s + p - c = 0 in columns 0..3, +1 elsewhere
            ent[c] = ent[S] + rel[0]
        else:         # subject replaced: c + p - o = 0 in columns 0..3, -1 elsewhere
            ent[c] = ent[O] - rel[0]
        ent[c, 4:] -= 1.0
    t = np.array([[S, 0, O]], np.int32)
    lp = {"margin": 16.0, "reduction": "sum"}  # every hinge active
    g_e, g_r, pads, got_loss = shared_step("TransE", k, eta, EDGE_E, 2, 1, "pairwise", lp, ent, rel, t, seed=seed)
    ref = _oracle("TransE", ent, rel, t, eta, seed, 1, "pairwise", lp)
    assert got_loss == ref.loss and pads
    assert torch.equal(g_e, ref.g_ent) and torch.equal(g_r, ref.g_rel)
    for row in [S, O] + cand[0].tolist():
        assert bool((g_e[row, :4] == 0).all()) and bool((g_e[row, 4:] != 0).all()), row
    assert bool((g_r[0, :4] == 0).all()) and bool((g_r[0, 4:] != 0).all())


def test_edge_rotate_zero_modulus():
    """RotatE with a theta = 0 relation row, where R(0) c - o and y - c are exactly 0 when the rows are equal: the
    reference's sqrt gradient is NaN there and rot_unit returns 0.  Chunk 0 (C = 2) is twice (A, 0, A') with A' = A and
    every candidate row = A: every residual is 0, so A, A' and the candidates get exactly 0, also in the second tile
    (gP = 0).  Chunk 1 is twice (Z, 0, Z') with Z' = Z in the first k/2 complex columns and every candidate row = Z:
    those columns of Z, Z', the candidates and the relation row's angle get exactly 0, the others of Z, Z' and the
    angle do not.  Chunk 2 is two ordinary positives.  The gradient is finite and within RotatEBound."""
    k, eta, C, B = 8, 40, 2, 6
    rels = np.array([0, 0, 0, 0, 1, 2])
    seed, cand, nk, free = _edge_seed(B, C, eta, rels, None, lambda c, s: bool((s[:, 2:4] == 0).any()))
    rng = np.random.default_rng(5)
    ent = xo.dyadic_table(rng, EDGE_E, 2 * k, frac_bits=2)
    rel = xo.dyadic_table(rng, 3, 2 * k, frac_bits=2)
    rel[0] = 0.0
    A, A1, Z, Z1, P0, P1, P2, P3 = free[:8]
    h = k // 2
    ent[A1] = ent[A]
    ent[Z] = 0.5
    ent[Z1] = ent[Z]
    ent[Z1, h:k] += 0.5
    ent[Z1, k + h:] -= 0.25
    ent[cand[0]] = ent[A]
    ent[cand[1]] = ent[Z]
    t = np.array([[A, 0, A1], [A, 0, A1], [Z, 0, Z1], [Z, 0, Z1], [P0, 1, P1], [P2, 2, P3]], np.int32)
    lp = {"margin": 3.0, "alpha": 0.5}
    g_e, g_r, pads, _ = shared_step("RotatE", k, eta, EDGE_E, 3, C, "self_adversarial", lp, ent, rel, t, seed=seed)
    ref = _oracle("RotatE", ent, rel, t, eta, seed, C, "self_adversarial", lp)
    for x in (g_e, g_r, ref.g_ent, ref.g_rel):
        assert bool(torch.isfinite(x).all())
    assert float(ref.sp[0]) == 0.0 and pads
    for row in [A, A1] + cand[0].tolist():
        assert bool((g_e[row] == 0).all()) and bool((ref.g_ent[row] == 0).all()), row
    zero_cols = np.r_[0:h, k:k + h]
    for row in [Z, Z1] + cand[1].tolist():
        assert bool((g_e[row, zero_cols] == 0).all()), row
    for row in (Z, Z1):
        assert bool((g_e[row, np.r_[h:k, k + h:2 * k]] != 0).all()), row
    assert bool((g_r[0, :h] == 0).all()) and bool((g_r[0, h:k] != 0).all())
    bound = xo.RotatEBound(ent, rel, t, ref, eta, loss="self_adversarial", loss_params=lp)
    for name, ok, ratio in bound.check(g_e, g_r, ref.g_ent, ref.g_rel):
        assert ok, (name, ratio)


# ---------------------------------------------------------------------------
# C = 1 is the per-positive step
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("model", ["TransE", "DistMult", "ComplEx", "HolE", "RotatE"])
@pytest.mark.parametrize("sampler", ["uniform", "bernoulli"])
def test_chunk_one_is_the_fused_step(model, sampler):
    from ampligraph_b200.datasets import negative_sampler_tables
    rng = _rng(model, sampler)
    E, R, B, eta, k = 150, 4, 60, 6, 32
    K = xo.internal_k(model, k)
    ent, rel = _glorot(rng, E, K), _glorot(rng, R, K)
    t = xo.zipf_triples(E, R, B, rng)
    loss, lp = "nll", {}
    tabs = negative_sampler_tables(t, E, R, "bernoulli") if sampler == "bernoulli" else None
    g_ent, g_rel, _, loss_s = shared_step(model, k, eta, E, R, 1, loss, lp, ent, rel, t, tabs)
    eng = _engine(model, k, eta, E, R, loss, lp)
    eng.set_embeddings(ent, rel)
    neg = None
    if tabs is not None:
        neg = eng.sample_negatives(_dev(t), NegativeSamplerTables(tabs, 1, eng.device), seed=SEED, step=STEP)
    eng.forward_backward(_dev(t), neg, seed=SEED, step=STEP)
    torch.cuda.synchronize()
    f_ent, f_rel = xo.dense(eng, eng.g_ent)[0], xo.dense(eng, eng.g_rel)[0]
    loss_f = eng.read_loss()
    eng.close()
    ne, nk = sno.sample(t, eta, E, SEED, STEP, 1, thresholds=tabs["thresholds"] if tabs is not None else None)
    kw = dict(rot_table=True) if model == "RotatE" else {}
    ref = xo.oracle_step(model, ent, rel, t, eta, ne, nk, loss=loss, loss_params=lp, device="cuda", **kw)
    bound = (xo.RotatEBound(ent, rel, t, ref, eta, loss, lp, device="cuda") if model == "RotatE"
             else xo.TrilinearBound(model, ent, rel, t, ref, eta, loss, lp, device="cuda"))
    for got_e, got_r in ((g_ent, g_rel), (f_ent, f_rel)):
        res = bound.check(got_e, got_r, ref.g_ent, ref.g_rel)
        assert all(ok for _, ok, _ in res), (model, sampler, res)
    for v in (loss_s, loss_f):
        assert abs(v - ref.loss) <= float(bound.loss_err) + 1e-12


# ---------------------------------------------------------------------------
# optimizers and the lazy rule
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("opt", ["sgd", "adam", "adagrad"])
@pytest.mark.parametrize("lazy", [False, True])
def test_optimizer_step_matches_injected(opt, lazy):
    """One shared step through apply_gradients(): its gradient is within TrilinearBound of the oracle on the same
    corruptions, and the per-positive step injected with those corruptions, given that gradient, leaves bit-identical
    tables, slots and stamps (the shared step stamps exactly the rows the per-positive step does).  Rows the step did
    not read keep their values, slots and stamps from before the step."""
    model, k, E, R, B, eta, C = "ComplEx", 16, 400, 5, 30, 8, 10
    rng = _rng(opt, lazy)
    K = xo.internal_k(model, k)
    ent, rel = _glorot(rng, E, K), _glorot(rng, R, K)
    t = xo.zipf_triples(E, R, B, rng)
    ne, nk = sno.sample(t, eta, E, SEED, STEP, C)
    out, grads = [], None
    for shared in (True, False):
        eng = _engine(model, k, eta, E, R, "nll", {}, optimizer=opt, optimizer_params={"learning_rate": 0.1},
                      lazy_tables=(lazy, lazy))
        eng.set_embeddings(ent, rel)
        state0 = [x.clone() for x in eng.slots["ent"] + eng.slots["rel"] if x is not None]
        if shared:
            eng.shared_negatives_backward(_dev(t), C, seed=SEED, step=STEP)
            grads = (eng.g_ent.clone(), eng.g_rel.clone())
        else:
            eng.forward_backward(_dev(t), (_dev(ne), _dev(nk)), seed=SEED, step=STEP)
            assert not eng._deferred
            eng.g_ent.copy_(grads[0])
            eng.g_rel.copy_(grads[1])
        eng.apply_gradients()
        torch.cuda.synchronize()
        e, r = eng.get_embeddings()
        stamps = [eng.stamps[key].cpu().clone() for key in ("ent", "rel")] if lazy else None
        slots = [x.cpu().clone() for x in eng.slots["ent"] + eng.slots["rel"] if x is not None]
        out.append((e.cpu(), r.cpu(), stamps, slots, [x.cpu() for x in state0]))
        if shared:
            ref = xo.oracle_step(model, ent, rel, t, eta, ne, nk, loss="nll", device="cuda")
            bound = xo.TrilinearBound(model, ent, rel, t, ref, eta, "nll", {}, device="cuda")
            res = bound.check(xo.dense(eng, grads[0])[0], xo.dense(eng, grads[1])[0], ref.g_ent, ref.g_rel)
            assert all(ok for _, ok, _ in res), res
        eng.close()
    (e1, r1, st1, sl1, init), (e2, r2, st2, sl2, _) = out
    assert torch.equal(e1, e2) and torch.equal(r1, r2)
    assert all(torch.equal(a, b) for a, b in zip(sl1, sl2))
    read = np.zeros(E, bool)
    read[t[:, 0]] = read[t[:, 2]] = True
    read[ne] = True
    unread = torch.as_tensor(~read)
    assert torch.equal(e1[unread], torch.as_tensor(ent)[unread])
    n_ent_slots = len(sl1) // 2
    for a, b in zip(sl1[:n_ent_slots], init[:n_ent_slots]):  # the entity slots of unread rows
        assert torch.equal(a[:E][unread], b[:E][unread])
    if lazy:
        assert all(torch.equal(a, b) for a, b in zip(st1, st2))
        stamp = int(_lib.load().kge_step_stamp(STEP))
        assert bool((st1[0][torch.as_tensor(read)] == stamp).all()) and bool((st1[0][unread] == 0).all())
        rel_read = np.zeros(R, bool)
        rel_read[t[:, 1]] = True
        assert bool((st1[1][torch.as_tensor(rel_read)] == stamp).all()) and bool((st1[1][torch.as_tensor(~rel_read)] == 0).all())


# ---------------------------------------------------------------------------
# end to end
# ---------------------------------------------------------------------------
def _structured(n=1500, E=200, R=4, seed=0):
    rng = np.random.default_rng(seed)
    s = rng.integers(0, E, n)
    p = rng.integers(0, R, n)
    o = (s * (p + 3) + p) % E
    return np.stack([s, p, o], 1).astype(np.int32)


@pytest.mark.parametrize("model", ["TransE", "DistMult", "ComplEx", "HolE", "RotatE"])
@pytest.mark.parametrize("reg", [None, "LP", "N3", "DURA"])
def test_fit_end_to_end(model, reg):
    from ampligraph_b200.latent_features import ScoringBasedEmbeddingModel, optimizers
    if reg in ("N3", "DURA") and model in ("TransE", "RotatE"):
        pytest.skip("compile refuses %s for %s" % (reg, model))
    x = _structured()

    def fit(reg, batch_size, epochs):
        m = ScoringBasedEmbeddingModel(eta=64, k=32, scoring_type=model, seed=3, max_ent_size=200, max_rel_size=4)
        m.data_indexer = False
        kw = {} if reg is None else {"entity_relation_regularizer": reg}
        m.compile(optimizer=optimizers.get("adam", {"learning_rate": 0.01}),
                  loss="self_adversarial" if model == "RotatE" else "multiclass_nll", **kw)
        m.fit(x, batch_size=batch_size, epochs=epochs, verbose=False, shared_negatives=16,
              negative_sampler="bernoulli" if model == "TransE" else "uniform")
        return m
    m = fit(reg, 300, 6)
    losses = m.history.history["loss"]
    assert np.isfinite(losses).all() and losses[-1] < losses[0], losses
    ranks = m.evaluate(x[:50], batch_size=50, verbose=False)
    assert len(ranks) == 50
    if reg is not None:
        # one step from the same tables: the same data term, plus the regulariser's
        with_reg, without = (fit(r, len(x), 1).history.history["loss"][0] for r in (reg, None))
        assert with_reg > without + 1e-9 * abs(without), (reg, with_reg, without)


# ---------------------------------------------------------------------------
# C ABI
# ---------------------------------------------------------------------------
def test_c_abi_refusals_and_sizer():
    import ctypes as C
    eng = _engine("DistMult", 8, 5, 50, 3, "pairwise", {})
    lib, h = eng.lib, eng.h
    for B in (0, 1, 7, 1000):
        for ch in (1, 3, 10 ** 6):
            assert lib.kge_shared_negatives_workspace_bytes(h, B, ch) == shared_negatives_workspace_bytes(B, 5)
    t = _dev(np.array([[0, 0, 1], [2, 1, 3]], np.int32))
    need = shared_negatives_workspace_bytes(2, 5)
    ws = torch.zeros(need // 4 + 64, dtype=torch.float32, device="cuda")
    P = lambda x: C.c_void_p(x.data_ptr()) if x is not None else None
    st = eng._stream()

    def call(chunk=2, B=2, ent=eng.ent, triples=t, wsb=need, sampler=None, w=ws, offset=0):
        wp = C.c_void_p(w.data_ptr() + offset) if w is not None else None
        return lib.kge_shared_negatives_step(h, chunk, P(ent), P(eng.rel), P(eng.g_ent), P(eng.g_rel), P(triples), B,
                                             sampler, 1, 2, P(eng.loss_acc), wp, wsb, st)
    assert call() == _lib.KGE_OK
    assert call(chunk=0) == _lib.KGE_ERR_INVALID_ARGUMENT
    assert call(B=-1) == _lib.KGE_ERR_INVALID_ARGUMENT
    assert call(B=(1 << 56) // 5 + 1) == _lib.KGE_ERR_INVALID_ARGUMENT
    assert call(ent=None) == _lib.KGE_ERR_INVALID_ARGUMENT
    assert call(triples=None) == _lib.KGE_ERR_INVALID_ARGUMENT
    assert call(wsb=need - 1) == _lib.KGE_ERR_INVALID_ARGUMENT
    assert call(B=0, ent=None, triples=None, w=None, wsb=0) == _lib.KGE_OK
    bad = _lib.KgeNegativeSampler(C.sizeof(_lib.KgeNegativeSampler) - 8, 1)
    assert call(sampler=C.byref(bad)) == _lib.KGE_ERR_INVALID_ARGUMENT
    bad = _lib.KgeNegativeSampler(C.sizeof(_lib.KgeNegativeSampler), 0)
    assert call(sampler=C.byref(bad)) == _lib.KGE_ERR_INVALID_ARGUMENT
    ids = torch.zeros(4, dtype=torch.int32, device="cuda")
    pooled = _lib.KgeNegativeSampler(C.sizeof(_lib.KgeNegativeSampler), 1)
    pooled.sub_pool_off, pooled.sub_pool_ids = ids.data_ptr(), ids.data_ptr()
    assert call(sampler=C.byref(pooled)) == _lib.KGE_ERR_UNSUPPORTED
    filt = _lib.KgeNegativeSampler(C.sizeof(_lib.KgeNegativeSampler), 1)
    filt.obj_filter_n, filt.obj_filter_keys, filt.obj_filter_vals = 1, ids.data_ptr(), ids.data_ptr()
    assert call(sampler=C.byref(filt)) == _lib.KGE_ERR_UNSUPPORTED
    stash = torch.zeros(64, dtype=torch.float32, device="cuda")
    _lib.check(lib.kge_set_row_stash(h, P(stash), 1))
    assert call() == _lib.KGE_ERR_UNSUPPORTED
    _lib.check(lib.kge_set_row_stash(h, None, 0))
    assert call() == _lib.KGE_OK
    assert call(offset=4) == _lib.KGE_ERR_INVALID_ARGUMENT  # workspace not 16-byte aligned
    _lib.check(lib.kge_set_embedding_dropout(h, 0.25, 0.0, 7))
    assert call() == _lib.KGE_ERR_UNSUPPORTED
    _lib.check(lib.kge_set_embedding_dropout(h, 0.0, 0.0, 0))
    # a pending deferred step (eta * B = 100 >= n_ent: the step buckets and defers)
    eng.forward_backward(_dev(np.tile(np.array([[1, 0, 2]], np.int32), (20, 1))), None, seed=0, step=0, defer=True)
    assert eng._deferred
    assert call() == _lib.KGE_ERR_INVALID_ARGUMENT
    eng.apply_gradients()
    assert call() == _lib.KGE_OK
    torch.cuda.synchronize()
    eng.close()
