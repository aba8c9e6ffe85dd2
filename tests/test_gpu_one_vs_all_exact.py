"""The 1vsAll family's kernels (kge_one_vs_all_step, kge_k_vs_all_step, kge_one_vs_all_relation_step; DESIGN.md 3.12
to 3.14) element by element against their float64 oracles, across the tile geometry of kge_train_1vsall.cu.

- Geometry sweep (bound tier): grid tables (exact logits) under exact_oracle.OvaBound, per element.  Each case asserts
  the geometry it claims: nsplit (candidate ranges of the stats and dQ passes), xsplit (query-tile ranges of the
  relation side's dX pass) and the number of 32-column chunks of a row.
- Bit-exact tier: gated tables on which every logit is exactly 0 or -128 (clipped), every live probability a power of
  two and so every fp32 operation exact: the gradient tables equal the oracle rounded to fp32.
- Clip edges: logits at -75 - 2^-4, -75, 75, 75 + 2^-4 and +-200 for all three objectives."""
import ctypes as C

import numpy as np
import pytest
import torch

import exact_oracle as xo
import k_vs_all_oracle
import one_vs_all_oracle
import relation_prediction_oracle
from ampligraph_b200 import _lib
from ampligraph_b200.engine import KGEEngine

pytestmark = pytest.mark.gpu


def _dev(a):
    return torch.as_tensor(a).cuda().contiguous()


def _grads(eng):
    out = []
    for g, rows in ((eng.g_ent, eng.ent_rows), (eng.g_rel, eng.n_rel)):
        d = torch.empty((rows, eng.internal_k), dtype=torch.float32, device=eng.device)
        _lib.check(eng.lib.kge_unpack_rows(eng.h, C.c_void_p(g.data_ptr()), C.c_void_p(d.data_ptr()), rows, eng._stream()))
        out.append(d.cpu().numpy())
    return out


def _csr(labels):
    off = np.concatenate([[0], np.cumsum([len(lab) for lab in labels])]).astype(np.int64)
    return off, np.concatenate(labels).astype(np.int32)


def _run(objective, model, k, ent, rel, q, side, reduction="sum", weight=1.0, labels=None, eps=0.0):
    """One step of `objective` ('ova' with side 's', 'o' or 's,o'; 'kva' with side 's' or 'o'; 'rel') on fresh
    gradient tables -> (loss, g_ent, g_rel) as float32 arrays of the dense [rows, internal_k] layout."""
    loss_name = "nll" if objective == "kva" else "multiclass_nll"
    eng = KGEEngine(model, k, 1, ent.shape[0], rel.shape[0], loss=loss_name, loss_params={"reduction": reduction},
                    optimizer="sgd")
    eng.set_embeddings(ent, rel)
    if objective == "ova":
        eng.one_vs_all_backward(_dev(q), side)
    elif objective == "kva":
        off, ids = _csr(labels)
        eng.k_vs_all_backward(_dev(q), side, _dev(off), _dev(ids), eps)
    else:
        eng.one_vs_all_relation_backward(_dev(q), weight)
    torch.cuda.synchronize()
    loss = float(eng.loss_acc[0])
    g_ent, g_rel = _grads(eng)
    eng.close()
    return loss, g_ent, g_rel


def _oracle(objective, model, ent, rel, q, side, reduction="sum", weight=1.0, labels=None, eps=0.0):
    if objective == "ova":
        return one_vs_all_oracle.loss_and_grads(model, ent, rel, q, side, reduction, matmul=True)
    if objective == "kva":
        return k_vs_all_oracle.loss_and_grads(model, ent, rel, q, labels, side, reduction, eps, matmul=True)
    return relation_prediction_oracle.loss_and_grads(model, ent, rel, q, weight, reduction, matmul=True)


def _bound_check(objective, model, k, ent, rel, q, side, reduction="sum", weight=1.0, labels=None, eps=0.0,
                 geometry=None):
    """Kernel against the oracle under OvaBound; geometry = (nsplit, xsplit, chunks) the case claims."""
    got_loss, g_ent, g_rel = _run(objective, model, k, ent, rel, q, side, reduction, weight, labels, eps)
    want_loss, want_ent, want_rel = _oracle(objective, model, ent, rel, q, side, reduction, weight, labels, eps)
    bound = xo.OvaBound(model, ent, rel, q)
    for sd in (["p"] if objective == "rel" else side.split(",")):
        ns, xs = bound.add_side(q, sd, reduction, weight, labels, eps)
    ld = xo.row_stride(model, ent.shape[1])
    if geometry is not None:
        assert (ns, xs, -(-ld // 32)) == geometry, ((ns, xs, -(-ld // 32)), geometry)
    where = (objective, model, k, side, reduction, eps)
    bound.check_loss(got_loss, want_loss, where)
    bound.check(g_ent, g_rel, want_ent, want_rel, where)
    return got_loss, g_ent, g_rel, want_ent, want_rel


def _triples(E, R, B, rng):
    t = np.stack([rng.integers(0, E, B), rng.integers(0, R, B), rng.integers(0, E, B)], 1).astype(np.int32)
    if B > 3:
        t[1] = t[0]
        t[2, 0] = t[2, 2]
    return t


def _labels(E, B, rng):
    """Labels on tile and split edges: 31/32, 63/64, the last entity, every entity, and a few random ones."""
    labels = [sorted(set(rng.integers(0, E, rng.integers(1, 6)).tolist())) for _ in range(B)]
    edges = [e for e in (0, 31, 32, 63, 64, 95, 96, E - 1) if e < E]
    labels[0] = edges
    if B > 1:
        labels[1] = list(range(E))
    if B > 2:
        labels[2] = [E - 1]
    return labels


def _queries(side, labels, E, R, rng):
    B = len(labels)
    keep, p = rng.integers(0, E, B), rng.integers(0, R, B)
    first = np.array([lab[0] for lab in labels])
    q = np.stack([keep, p, first], 1) if side == "o" else np.stack([first, p, keep], 1)
    return q.astype(np.int32)


# --------------------------------------------------------------------------
# (a) geometry sweep on grid tables, per-element bound
# --------------------------------------------------------------------------
# (id, objective, model, k, n_ent, n_rel, B, (nsplit, xsplit, chunks)): nsplit / xsplit from the kernel's rule
SWEEP = [
    ("ld32-one-chunk", "ova", "DistMult", 32, 300, 5, 100, (10, 1, 1)),
    ("ld36-zero-filled-tail", "ova", "DistMult", 36, 300, 5, 100, (10, 1, 2)),
    ("ld80-three-chunks", "ova", "DistMult", 80, 300, 5, 100, (10, 1, 3)),
    ("complex-kp36-imag-in-chunk", "ova", "ComplEx", 36, 300, 5, 100, (10, 1, 3)),
    ("complex-kp52-imag-in-chunk", "ova", "ComplEx", 52, 300, 5, 100, (10, 1, 4)),
    ("hole-k64", "ova", "HolE", 64, 300, 5, 100, (10, 1, 4)),
    ("nsplit64-uneven", "ova", "DistMult", 12, 2100, 5, 40, (64, 1, 1)),
    ("nsplit-capped-by-tiles", "ova", "ComplEx", 10, 100, 5, 40, (4, 1, 1)),
    ("nsplit7-uneven", "ova", "DistMult", 16, 640, 5, 1280, (7, 1, 1)),
    ("nsplit1-8500", "ova", "DistMult", 8, 300, 5, 8500, (1, 1, 1)),
    ("B1", "ova", "ComplEx", 10, 45, 3, 1, (2, 1, 1)),
    ("n_ent2", "ova", "DistMult", 8, 2, 3, 50, (1, 1, 1)),
    ("n_ent-off-grid", "ova", "HolE", 16, 1007, 3, 70, (32, 1, 1)),
    ("rel-xsplit1", "rel", "DistMult", 36, 50, 300, 32, (10, 1, 2)),
    ("rel-xsplit", "rel", "ComplEx", 36, 50, 45, 200, (2, 7, 3)),
    ("rel-nsplit64", "rel", "DistMult", 12, 50, 2100, 40, (64, 2, 1)),
    ("rel-n_rel2", "rel", "HolE", 16, 50, 2, 70, (1, 3, 1)),
    ("rel-B1", "rel", "DistMult", 8, 50, 45, 1, (2, 1, 1)),
    ("kva-nsplit64", "kva", "DistMult", 12, 2100, 5, 40, (64, 1, 1)),
    ("kva-complex-kp52", "kva", "ComplEx", 52, 300, 5, 100, (10, 1, 4)),
    ("kva-n_ent2", "kva", "HolE", 16, 2, 3, 33, (1, 1, 1)),
    ("kva-B1", "kva", "DistMult", 36, 1007, 3, 1, (32, 1, 2)),
]


@pytest.mark.parametrize("reduction", ["sum", "mean"])
@pytest.mark.parametrize("case", SWEEP, ids=[c[0] for c in SWEEP])
def test_geometry_sweep(case, reduction):
    _, objective, model, k, E, R, B, geometry = case
    rng = np.random.default_rng(k * 7919 + E + B)
    K = xo.internal_k(model, k)
    ent, rel = xo.grid_table(rng, E, K), xo.grid_table(rng, R, K)
    if objective == "kva":
        for side, eps in (("o", 0.0), ("s", 0.1)):
            labels = _labels(E, B, rng)
            q = _queries(side, labels, E, R, rng)
            _bound_check("kva", model, k, ent, rel, q, side, reduction, labels=labels, eps=eps, geometry=geometry)
    elif objective == "rel":
        _bound_check("rel", model, k, ent, rel, _triples(E, R, B, rng), None, reduction, weight=0.5, geometry=geometry)
    else:
        _bound_check("ova", model, k, ent, rel, _triples(E, R, B, rng), "s,o", reduction, geometry=geometry)


def _largest_ld(extra_bytes):
    """The largest row stride (a multiple of 4 floats) whose [32, ld] accumulator, staging buffers and g tile fit the
    device's opt-in shared memory per block (kge_train_1vsall.cu, one_vs_all_smem_bytes)."""
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    fixed = (4 * 32 * 36 + 32 * 33) * 4 + extra_bytes
    return (optin - fixed) // (32 * 4) // 4 * 4


@pytest.mark.parametrize("objective", ["ova", "kva", "rel"])
def test_largest_accepted_row_and_the_next_refused(objective):
    """DistMult at the largest ld the shared-memory check accepts (the [32, ld] accumulator at the opt-in limit) runs and
    meets the bound; ld + 4 is refused with KGE_ERR_UNSUPPORTED (NotImplementedError)."""
    ld = _largest_ld(32 * 4 if objective == "kva" else 0)
    rng = np.random.default_rng(ld)
    E, R, B = 70, 40, 40
    ent = xo.grid_table(rng, E, ld, values=[-0.5, 0.0, 0.5])
    rel = xo.grid_table(rng, R, ld, values=[-0.5, 0.0, 0.5])
    if objective == "kva":
        labels = _labels(E, B, rng)
        _bound_check("kva", "DistMult", ld, ent, rel, _queries("o", labels, E, R, rng), "o", labels=labels, eps=0.1)
    elif objective == "rel":
        _bound_check("rel", "DistMult", ld, ent, rel, _triples(E, R, B, rng), None)
    else:
        _bound_check("ova", "DistMult", ld, ent, rel, _triples(E, R, B, rng), "s,o")
    k = ld + 4
    eng = KGEEngine("DistMult", k, 1, E, R, loss="nll" if objective == "kva" else "multiclass_nll")
    t = _dev(_triples(E, R, B, rng))
    with pytest.raises(NotImplementedError, match="shared-memory"):
        if objective == "kva":
            off, ids = _csr(_labels(E, B, rng))
            eng.k_vs_all_backward(t, "o", _dev(off), _dev(ids))
        elif objective == "rel":
            eng.one_vs_all_relation_backward(t, 1.0)
        else:
            eng.one_vs_all_backward(t, "s,o")
    eng.close()


# --------------------------------------------------------------------------
# (b) bit-exact tier: gated tables
# --------------------------------------------------------------------------
def exact_value(want):
    """The float64 oracle snapped to multiples of 2^-40 of its largest entry, as float32: on the gated tables every
    true value is such a multiple and fp32-exact, and the oracle's own residue (torch's logsumexp backward forms
    exp(l - log D), with log D rounded) is far below that unit."""
    want = np.asarray(want, np.float64)
    top = np.abs(want).max()
    if top == 0:
        return want.astype(np.float32)
    unit = 2.0 ** (np.ceil(np.log2(top)) - 40)
    return (np.round(want / unit) * unit).astype(np.float32)


def gated_tables(model, k, G, group, R, rng, rel_live=None):
    """Entity e one-hot on gate column group[e] of [0, G) (the real half for ComplEx), grid noise on the columns past the
    gates (ComplEx: of the imaginary half) and 0 elsewhere.  Relation rows: -128 on every gate and 0 elsewhere; with
    rel_live[r] (a set of groups), 0 on the gates of those groups and grid noise past the gates (the relation side's
    candidates).  Every logit f(s, p, x) of a same-group pair is then -128, every other exactly 0."""
    K = xo.internal_k(model, k)
    E = len(group)
    noise_lo, noise_hi = (G, k) if model == "DistMult" else (k + G, 2 * k)
    ent = np.zeros((E, K), np.float32)
    ent[np.arange(E), group] = 1.0
    ent[:, noise_lo:noise_hi] = xo.grid_table(rng, E, noise_hi - noise_lo)
    rel = np.zeros((R, K), np.float32)
    rel[:, :G] = -128.0
    if rel_live is not None:
        for r, live in enumerate(rel_live):
            rel[r, sorted(live)] = 0.0
    return ent, rel


def _exact_ova_case(model, k, G, g, B, R, rng):
    """n_ent = G g with (G - 1) g a power of two; targets outside the kept entity's group, so each row has (G - 1) g
    live candidates."""
    group = np.repeat(np.arange(G), g)
    E = G * g
    s = rng.integers(0, E, B)
    o = (s + g * rng.integers(1, G, B)) % E  # another group
    t = np.stack([s, rng.integers(0, R, B), o], 1).astype(np.int32)
    ent, rel = gated_tables(model, k, G, group, R, rng)
    return ent, rel, t


# (model, k, G, g, B): n_ent = G g; (G - 1) g = 2^j live candidates per row
EXACT_OVA = [("DistMult", 36, 5, 16, 100), ("DistMult", 80, 65, 16, 300), ("DistMult", 80, 65, 32, 40),
             ("DistMult", 36, 5, 16, 8500), ("ComplEx", 36, 5, 16, 100), ("ComplEx", 80, 17, 64, 150)]


@pytest.mark.parametrize("case", EXACT_OVA, ids=["-".join(map(str, c)) for c in EXACT_OVA])
def test_bit_exact_one_vs_all(case):
    model, k, G, g, B = case
    rng = np.random.default_rng(G * g + B)
    ent, rel, t = _exact_ova_case(model, k, G, g, B, 4, rng)
    live = (G - 1) * g
    assert live & (live - 1) == 0
    loss, g_ent, g_rel = _run("ova", model, k, ent, rel, t, "s,o")
    want_loss, want_ent, want_rel = one_vs_all_oracle.loss_and_grads(model, ent, rel, t, "s,o", "sum", matmul=True)
    assert np.array_equal(g_ent, exact_value(want_ent)), np.abs(g_ent - want_ent).max()
    assert np.array_equal(g_rel, exact_value(want_rel)), np.abs(g_rel - want_rel).max()
    assert want_loss == pytest.approx(2 * B * np.log(live), rel=1e-12)
    assert loss == pytest.approx(want_loss, rel=1e-6)


# (model, k, G, g, B, reduction, eps): n_ent = G g, a power of two under mean or eps > 0 (eps = 1/2: y' dyadic)
EXACT_KVA = [("DistMult", 36, 5, 16, 100, "sum", 0.0), ("DistMult", 80, 64, 32, 40, "mean", 0.0),
             ("DistMult", 36, 8, 16, 300, "sum", 0.5), ("ComplEx", 36, 4, 16, 100, "mean", 0.5),
             ("ComplEx", 36, 7, 10, 70, "sum", 0.0)]


@pytest.mark.parametrize("side", ["o", "s"])
@pytest.mark.parametrize("case", EXACT_KVA, ids=["-".join(map(str, c)) for c in EXACT_KVA])
def test_bit_exact_k_vs_all(case, side):
    """Live sigmoid 1/2: g = w (1/2 - y') is dyadic for any labels (also dead or on tile edges)."""
    model, k, G, g, B, reduction, eps = case
    rng = np.random.default_rng(G * g + B)
    group = np.repeat(np.arange(G), g)
    E = G * g
    ent, rel = gated_tables(model, k, G, group, 4, rng)
    labels = _labels(E, B, rng)
    q = _queries(side, labels, E, 4, rng)
    _, g_ent, g_rel = _run("kva", model, k, ent, rel, q, side, reduction, labels=labels, eps=eps)
    _, want_ent, want_rel = k_vs_all_oracle.loss_and_grads(model, ent, rel, q, labels, side, reduction, eps,
                                                           matmul=True)
    assert np.array_equal(g_ent, exact_value(want_ent)), np.abs(g_ent - want_ent).max()
    assert np.array_equal(g_rel, exact_value(want_rel)), np.abs(g_rel - want_rel).max()


def exact_relation_case(model, k, B, rng, n_live=4, G=2, g=16):
    """Relation side: G groups of g entities; relation r is live (0 on the gate) for group r // n_live only, so every
    (s, o) pair of one group has n_live live relations, among them its own p."""
    group = np.repeat(np.arange(G), g)
    R = G * n_live
    ent, rel = gated_tables(model, k, G, group, R, rng, [{r // n_live} for r in range(R)])
    gs = rng.integers(0, G, B)
    s, o = gs * g + rng.integers(0, g, B), gs * g + rng.integers(0, g, B)
    p = gs * n_live + rng.integers(0, n_live, B)
    return ent, rel, np.stack([s, p, o], 1).astype(np.int32)


# (model, k, B, live relations per group, groups): B <= 32 (xsplit 1) and above
EXACT_REL = [("DistMult", 36, 32, 4, 2), ("DistMult", 36, 300, 8, 9), ("ComplEx", 36, 200, 4, 5),
             ("ComplEx", 12, 1000, 2, 3)]


@pytest.mark.parametrize("model,k,B,n_live,G", EXACT_REL)
def test_bit_exact_relation_side(model, k, B, n_live, G):
    rng = np.random.default_rng(B + n_live)
    ent, rel, t = exact_relation_case(model, k, B, rng, n_live, G)
    loss, g_ent, g_rel = _run("rel", model, k, ent, rel, t, None, weight=0.5)
    want_loss, want_ent, want_rel = relation_prediction_oracle.loss_and_grads(model, ent, rel, t, 0.5, matmul=True)
    assert np.array_equal(g_ent, exact_value(want_ent)), np.abs(g_ent - want_ent).max()
    assert np.array_equal(g_rel, exact_value(want_rel)), np.abs(g_rel - want_rel).max()
    assert want_loss == pytest.approx(0.5 * B * np.log(n_live), rel=1e-12)
    assert loss == pytest.approx(want_loss, rel=1e-6)


# --------------------------------------------------------------------------
# (c) clip edges
# --------------------------------------------------------------------------
CLIP_TARGETS = [-75.0 - 2.0 ** -4, -75.0, 75.0, 75.0 + 2.0 ** -4, 200.0, -200.0]


def clip_tables():
    """DistMult k = 8.  Entities: 0 = ones, 1 = -ones, 2 = zeros (the target), 3 + i = X_i with CLIP_TARGETS[i] / 8 in
    every column.  Relations: 0 = ones (the positives'), 1 + i = X_i as well (the relation side's candidates).  The two
    positives (0, 0, 2) and (1, 0, 2) give X_i the logits +-CLIP_TARGETS[i] on side o and on side p (s = +-ones,
    o = ones there): X_i is fed by those two logits only, both clipped unless |CLIP_TARGETS[i]| = 75."""
    n = len(CLIP_TARGETS)
    ent = np.zeros((3 + n, 8), np.float32)
    ent[0], ent[1] = 1.0, -1.0
    rel = np.zeros((1 + n, 8), np.float32)
    rel[0] = 1.0
    for i, v in enumerate(CLIP_TARGETS):
        ent[3 + i] = rel[1 + i] = v / 8.0
    return ent, rel


@pytest.mark.parametrize("reduction", ["sum", "mean"])
@pytest.mark.parametrize("objective", ["ova", "kva", "rel"])
def test_clip_edges(objective, reduction):
    """Rows fed only by clipped logits are exactly 0 in the kernel and the oracle; rows with a logit at exactly +-75
    are not; everything meets the bound."""
    ent, rel = clip_tables()
    if objective == "rel":
        t = np.array([[0, 0, 0], [1, 0, 0]], np.int32)  # s = +-ones, o = ones: Qp = +-ones
        _, g_ent, g_rel, want_ent, want_rel = _bound_check("rel", "DistMult", 8, ent, rel, t, None, reduction)
        got, want, first = g_rel, want_rel, 1
    else:
        t = np.array([[0, 0, 2], [1, 0, 2]], np.int32)
        labels = [[2], [2]] if objective == "kva" else None
        _, g_ent, g_rel, want_ent, want_rel = _bound_check(objective, "DistMult", 8, ent, rel, t, "o", reduction,
                                                           labels=labels)
        got, want, first = g_ent, want_ent, 3
    for i, v in enumerate(CLIP_TARGETS):
        row = first + i
        if abs(v) > 75.0:
            assert (want[row] == 0).all() and (got[row] == 0).all(), (objective, v, got[row])
        else:
            assert (want[row] != 0).all() and (got[row] != 0).all(), (objective, v, got[row], want[row])
