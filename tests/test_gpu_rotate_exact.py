"""RotatE training element by element: every element of g_ent, g_rel, the scores and the loss of one step against the
float64 oracle on the kernels' rotation table, within exact_oracle.RotatEBound (derived in its docstring), on the fast
path (kge_train_rot_kernel) and the general kernel's RotatE Scorer.

Each case asserts the kernel it targets ran (the launched kernel's name, from torch.profiler), holds the exact
properties with no tolerance (the relation rows' second halves, every pad column and every row no term touches are 0),
prints its worst error / bound ratio, and shows the check is sensitive on the device: the kernel's output fails it
against the oracle with one corruption's term removed."""
import zlib

import numpy as np
import pytest
import torch

import exact_oracle as xo
from ampligraph_b200 import _lib

pytestmark = pytest.mark.gpu


def _seed(*a):
    return zlib.crc32(repr(a).encode())


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a)).cuda().contiguous()


def _force(monkeypatch, **env):
    for var in ("KGE_B200_TRAIN_KERNEL", "KGE_B200_TRAIN_SCHED", "KGE_B200_TRAIN_NBUF", "KGE_B200_ROT_G"):
        monkeypatch.delenv(var, raising=False)
    for var, val in env.items():
        if val is not None:
            monkeypatch.setenv(var, str(val))


def rot_group(k, eta, forced=None):
    """The fast path's group size by kge_create's rule (kge_api.cu): cap rows per warp beside 8 warps; all eta when they
    fit, else cap / 2; KGE_B200_ROT_G = g is taken when 1 <= g <= cap / 2 and g < eta."""
    max_smem = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    kp = -(-k // 4) * 4
    eta_pad = -(-eta // 4) * 4
    rot_aux = (4 * eta_pad * 4 + 16 + 15) // 16 * 16
    cap = (max_smem // 8 - rot_aux) // (2 * kp * 4)
    G = eta if cap >= eta else cap // 2
    if forced is not None and 1 <= forced <= cap // 2 and forced < eta:
        G = forced
    return G


def _sides(rng, eta, B, n0):
    """keep flags [eta*B] (1: object replaced) with n0 subject-replaced corruptions per positive (None: random)."""
    if n0 is None:
        return rng.integers(0, 2, eta * B).astype(np.uint8)
    nk = np.ones((eta, B), np.uint8)
    for i in range(B):
        nk[rng.permutation(eta)[:n0], i] = 0
    return nk.reshape(-1)


def _tables(rng, E, R, k, edge):
    K = 2 * k
    ent = rng.uniform(-1, 1, (E, K)).astype(np.float32)
    rel = rng.uniform(-1, 1, (R, K)).astype(np.float32)
    div, _ = xo.rotation_divisor32(K, R)
    if edge == "tiny":      # |v|^2 in [2^-126, 1e-30): rot_unit's clamp must not apply
        ent *= np.float32(2.0 ** -56)
    elif edge == "huge":    # |v|^2 up to 2^127, below FLT_MAX
        ent *= np.float32(2.0 ** 62)
    elif edge == "angles":  # theta = 0 (c = 1, sn = 0 exactly) and |phi| up to 1e4 rad
        rel[0] = 0.0
        rel[1:] = (rng.uniform(-1e4, 1e4, (R - 1, K)) * float(div)).astype(np.float32)
    return ent, rel


def run_case(monkeypatch, k, eta, *, E=2000, R=11, B=300, mode="ext", loss="self_adversarial", lp=None, path="rot",
             env=None, neg_group=0, stash=False, negatives="injected", n0=None, edge=None, seed=0):
    """One step; every element checked against RotatEBound.  path 'rot' / 'general': the kernel that must have run."""
    rng = np.random.default_rng(_seed(k, eta, E, B, mode, loss, str(lp), path, str(env), neg_group, stash, negatives,
                                      n0, edge, seed))
    env = dict(env or {})
    if path == "general":
        env["KGE_B200_TRAIN_KERNEL"] = "general"
    _force(monkeypatch, **env)
    from ampligraph_b200.engine import KGEEngine
    lp = dict(lp or {})
    ent, rel = _tables(rng, E, R, k, edge)
    t = xo.zipf_triples(E, R, B, rng)
    if edge == "near_zero":  # o = R(phi) s up to an ulp for the first positive: its residual is ~1e-8
        h = k
        div, _ = xo.rotation_divisor32(2 * k, R)
        c, s = xo.rotation_table(rel[t[0, 1], :h], div)
        sr, si = ent[t[0, 0], :h], ent[t[0, 0], h:]
        yr = (np.float64(-si) * s + np.float64(sr * c)).astype(np.float32)
        yi = (np.float64(sr) * s + np.float64(si * c)).astype(np.float32)
        if t[0, 2] == t[0, 0]:
            t[0, 2] = (t[0, 0] + 1) % E
        ent[t[0, 2], :h], ent[t[0, 2], h:] = np.nextafter(yr, np.float32(2)), yi
    eng = KGEEngine("RotatE", k, eta, E, R, loss=loss, loss_params=lp, neg_group=neg_group)
    if stash:
        st = eng.ensure_row_stash(B)
        assert st is not None, "expected a geometry that stashes"
        st.fill_(float("nan"))
    eng.set_embeddings(ent, rel)
    sp = torch.full((B,), float("nan"), device="cuda")
    sn = torch.full((eta * B,), float("nan"), device="cuda")
    if negatives == "philox":
        seed_, step_ = 7, 2
        corr = eng.generate_corruptions(_dev(t), seed=seed_, step=step_).cpu().numpy()
        neg, ne, nk = None, corr, None
    else:
        ne = rng.integers(0, E, eta * B).astype(np.int32)
        nk = _sides(rng, eta, B, n0)
        same = rng.random(eta * B) < 0.03  # N = P: the replaced entity is the one it replaces
        tiled = np.tile(t, (eta, 1))
        ne[same] = np.where(nk[same] == 1, tiled[same, 2], tiled[same, 0])
        seed_, step_, neg = 0, 0, (_dev(ne), _dev(nk))
    ext = {}
    kw = dict(seed=seed_, step=step_)
    if mode == "ext":
        ext = dict(dpos=rng.uniform(-1, 1, B).astype(np.float32), dneg=rng.uniform(-1, 1, eta * B).astype(np.float32))
        kw.update(mode=_lib.STEP_BACKWARD_EXT, dpos=_dev(ext["dpos"]), dneg=_dev(ext["dneg"]))
    else:
        kw.update(mode=_lib.STEP_FORWARD_ONLY if mode == "forward" else _lib.STEP_FUSED, scores_pos=sp, scores_neg=sn)
    names = xo.launched(lambda: eng.forward_backward(_dev(t), neg, **kw))
    g_ent, ent_pads = xo.dense(eng, eng.g_ent)
    g_rel, rel_pads = xo.dense(eng, eng.g_rel)
    got_loss = eng.read_loss()
    for _ in range(3):  # a short profiling session now and then records no kernel at all: replay the step's scores
        if names:       # (FORWARD_ONLY into scratch buffers: the same kernel choice, nothing the checks read is written)
            break
        names = xo.launched(lambda: eng.forward_backward(
            _dev(t), neg, seed=seed_, step=step_, mode=_lib.STEP_FORWARD_ONLY,
            scores_pos=torch.empty(B, device="cuda"), scores_neg=torch.empty(eta * B, device="cuda")))
    eng.close()
    where = "k=%d eta=%d %s %s %s env=%s edge=%s" % (k, eta, path, mode, loss, env, edge)

    # the kernel that ran
    nch = -(-min(-(-k // 4) * 4, 512 if path == "general" else 10 ** 9) // 4)  # float4 chunks per (window) half
    nit = 1 if nch <= 32 else 2 if nch <= 64 else 4
    want_kernel = "kge_train_rot_kernel<%d>" % nit if path == "rot" else "kge_train_kernel<4, %d" % nit
    assert any(want_kernel in n for n in names), (where, sorted(names))
    if path == "rot" and "KGE_B200_ROT_G" in env:
        assert rot_group(k, eta, int(env["KGE_B200_ROT_G"])) == int(env["KGE_B200_ROT_G"]), where

    ref = xo.oracle_step("RotatE", ent, rel, t, eta, ne, nk, loss=loss, loss_params=lp, rot_table=True,
                         max_rel_size=R, **ext)
    bound = xo.RotatEBound(ent, rel, t, ref, eta, loss=None if mode in ("ext", "forward") else loss, loss_params=lp,
                           max_rel_size=R)
    ratios = {}
    if mode != "ext":
        for name, got, want in (("sp", sp, ref.sp), ("sn", sn, ref.sn)):
            ok, ratios[name] = bound.check_scores(got.cpu().double(), want, name)
            assert ok, (where, name, ratios[name])
    if mode == "forward":
        assert bool((g_ent == 0).all()) and bool((g_rel == 0).all()), where
        print("\n%s: worst error / bound %s" % (where, ratios))
        return
    if mode == "fused":
        assert abs(got_loss - ref.loss) <= bound.loss_err, (where, got_loss, ref.loss, bound.loss_err)
    res = bound.check(g_ent, g_rel, ref.g_ent, ref.g_rel)
    for name, ok, r in res:
        ratios[name] = r
        assert ok, (where, name, "worst error / bound %.3g" % r)
    print("\n%s: worst error / bound %s" % (where, {n: round(r, 4) for n, r in ratios.items()}))

    # exact properties
    assert ent_pads and rel_pads, where + ": gradient pad columns written"
    assert bool((g_rel[:, k:] == 0).all()), where + ": second half of a relation row"
    corr = ref.corr.numpy()
    touched_e = np.zeros(E, bool)
    touched_e[np.concatenate([t[:, 0], t[:, 2], corr[:, 0], corr[:, 2]])] = True
    touched_r = np.zeros(R, bool)
    touched_r[t[:, 1]] = True
    assert bool((g_ent[~touched_e] == 0).all()) and bool((g_rel[~touched_r] == 0).all()), where + ": untouched rows"

    # sensitivity: the check rejects the kernel's output against the oracle without one corruption whose replaced
    # entity occurs once in the step
    lookups = np.bincount(np.concatenate([t[:, 0], t[:, 2], corr[:, 0], corr[:, 2]]), minlength=E)
    repl = np.where(corr[:, 0] != np.tile(t[:, 0], eta), corr[:, 0], corr[:, 2])
    cands = [r for r in np.nonzero(lookups[repl] == 1)[0] if float(ref.dsn[r]) != 0.0]
    assert cands, where + ": no corruption with a replaced entity of its own"
    r = int(cands[0])
    i = r % B
    keep = int(corr[r, 0] == t[i, 0] and corr[r, 2] != t[i, 2]) if nk is None else int(nk[r])
    one = xo.oracle_step("RotatE", ent, rel, t[i:i + 1], 1, [repl[r]], [keep], dpos=[0.0], dneg=[float(ref.dsn[r])],
                         rot_table=True, max_rel_size=R)
    res = bound.check(g_ent, g_rel, ref.g_ent - one.g_ent, ref.g_rel - one.g_rel)
    assert not all(ok for _, ok, _ in res), where + ": the check accepts a dropped corruption"


# ---------------------------------------------------------------------------
# the fast path: NIT = 1 and 2, groups, eta, sides
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("k", [20, 50, 128, 129, 200, 256])
def test_fast_path_row_shapes(k, monkeypatch):
    """NIT = 1 (k = 20; 50: pad columns, nch = 13; 128) and NIT = 2 (129: one live lane in the second chunk; 200; 256),
    everything resident."""
    run_case(monkeypatch, k, 7)
    assert rot_group(k, 7) == 7


FAST_GROUPS = [(64, 7, 2, None), (64, 10, 3, 3), (64, 23, 5, None), (64, 9, 3, 3), (64, 9, 3, 4), (64, 9, None, 9),
               (64, 9, None, 0), (64, 1, None, None), (64, 9, None, None), (64, 40, None, 17), (64, 40, 7, 13),
               (200, 30, None, None)]


@pytest.mark.parametrize("k,eta,G,n0", FAST_GROUPS)
def test_fast_path_groups_and_sides(k, eta, G, n0, monkeypatch):
    """KGE_B200_ROT_G forcing 2, 3 and 5 (2 to 5+ groups, short last groups); eta = 1, odd, > 32 (two ballot rounds);
    all corruptions on the subject side (n0 = eta), all on the object side (n0 = 0), n0 at a group boundary (3 with
    G = 3) and inside one (4); odd side counts run the self-paired last row in both loops."""
    run_case(monkeypatch, k, eta, env={"KGE_B200_ROT_G": G} if G else None, n0=n0)


# ---------------------------------------------------------------------------
# the general kernel's RotatE Scorer
# ---------------------------------------------------------------------------
GENERAL = [dict(k=64, eta=9, n0=3), dict(k=64, eta=9, n0=0), dict(k=64, eta=40, n0=17), dict(k=129, eta=7),
           dict(k=700, eta=5),                              # column windows
           dict(k=64, eta=9, neg_group=1), dict(k=64, eta=10, neg_group=3, n0=3),
           dict(k=64, eta=10, neg_group=3, env={"KGE_B200_TRAIN_NBUF": 1}),
           dict(k=64, eta=10, neg_group=3, stash=True), dict(k=700, eta=5, neg_group=2, stash=True),
           dict(k=64, eta=9, env={"KGE_B200_TRAIN_SCHED": "dynamic"})]


@pytest.mark.parametrize("case", GENERAL, ids=lambda c: "-".join("%s%s" % kv for kv in sorted(c.items())))
def test_general_kernel(case, monkeypatch):
    case = dict(case)
    run_case(monkeypatch, case.pop("k"), case.pop("eta"), path="general", **case)


# ---------------------------------------------------------------------------
# modes, losses, negatives
# ---------------------------------------------------------------------------
LOSSES = [("self_adversarial", {"margin": 3.0, "alpha": 0.5}), ("self_adversarial", {"reduction": "mean"}),
          ("nll", {}), ("multiclass_nll", {}), ("pairwise", {"margin": 0.37}),
          ("absolute_margin", {"margin": 33.0})]  # scores near -33 (k = 32): about half the hinges active


@pytest.mark.parametrize("path", ["rot", "general"])
@pytest.mark.parametrize("loss,lp", LOSSES, ids=["%s-%s" % (l, p.get("reduction", "sum")) for l, p in LOSSES])
def test_fused_losses(loss, lp, path, monkeypatch):
    """The fused step: dL/dscore from the kernel's own scores, within the score bound propagated through each
    positive's loss Hessian; the hinge losses under the premise that no hinge argument is within its bound of 0."""
    run_case(monkeypatch, 32, 9, mode="fused", loss=loss, lp=lp, path=path, B=200, E=2000, R=5)


@pytest.mark.parametrize("path", ["rot", "general"])
@pytest.mark.parametrize("mode,negatives", [("forward", "injected"), ("ext", "philox"), ("fused", "philox")])
def test_modes_and_philox(mode, negatives, path, monkeypatch):
    """FORWARD_ONLY (scores only, gradients untouched) and the Philox draw replayed with generate_corruptions."""
    run_case(monkeypatch, 50, 8, mode=mode, negatives=negatives, path=path)


# ---------------------------------------------------------------------------
# edges
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("path", ["rot", "general"])
@pytest.mark.parametrize("edge", ["tiny", "huge", "angles", "near_zero"])
def test_edges(edge, path, monkeypatch):
    """Rows scaled by 2^-56 (|v|^2 in [2^-126, 1e-30): each unit vector must be g v / |v|, not g v 1e15), rows near
    2^62 (|v|^2 up to 2^127), theta = 0 and |phi| up to 1e4 rad, and a residual of ~1e-8 (o = R(phi) s up to an ulp)."""
    run_case(monkeypatch, 40, 7, edge=edge, path=path)
