"""GPU parity tests: the CUDA path (through the C-ABI) against the oracle.

Run on an H100 with `pytest -m gpu`.  Tolerances: fp32 scores / gradients /
losses within 1e-4 relative (BASELINE.json north_star); ranks bit-exact.
"""
import zlib

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

MODELS = ["TransE", "DistMult", "ComplEx", "HolE", "RotatE"]
LOSSES = ["pairwise", "nll", "absolute_margin", "self_adversarial", "multiclass_nll"]
RTOL = 1e-4


def _engine(*a, **kw):
    from ampligraph_b200.engine import KGEEngine
    return KGEEngine(*a, **kw)


def _tables(model, E, R, k, rng, scale=None):
    K = k if model in ("TransE", "DistMult") else 2 * k
    lim_e = scale or np.sqrt(6.0 / (E + K))
    lim_r = scale or np.sqrt(6.0 / (R + K))
    ent = rng.uniform(-lim_e, lim_e, (E, K)).astype(np.float32)
    rel = rng.uniform(-lim_r, lim_r, (R, K)).astype(np.float32)
    return ent, rel


def _triples(E, R, n, rng):
    return np.stack([rng.integers(0, E, n), rng.integers(0, R, n), rng.integers(0, E, n)], 1).astype(np.int32)


def _negatives(E, B, eta, rng):
    return rng.integers(0, E, B * eta).astype(np.int32), rng.integers(0, 2, B * eta).astype(np.uint8)


def _dev(a):
    return torch.as_tensor(a).cuda().contiguous()


def _dense(eng, table):
    """padded [rows, ld] -> dense [rows, internal_k] (host-side slicing, independent of kge_unpack_rows)."""
    t = table.detach().cpu().numpy()
    k, kp = eng.k, eng.kp
    if eng.internal_k == k:
        return t[:, :k].copy()
    return np.concatenate([t[:, :k], t[:, kp:kp + k]], axis=1)


def _close(a, b, rtol=RTOL):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    scale = max(np.abs(b).max(), 1e-30)
    return np.abs(a - b).max() <= rtol * scale + 1e-7


# ---------------------------------------------------------------------------
def test_library_loads_and_layout():
    from ampligraph_b200 import _lib
    lib = _lib.load()
    assert lib.kge_abi_version() == _lib.ABI_VERSION
    for model, k, ld in (("TransE", 50, 52), ("DistMult", 400, 400), ("ComplEx", 3, 8), ("RotatE", 200, 400)):
        eng = _engine(model, k, 2, 10, 3)
        assert eng.ld == ld and eng.internal_k == (k if model in ("TransE", "DistMult") else 2 * k)
        eng.close()


@pytest.mark.parametrize("model", MODELS)
def test_pack_unpack_roundtrip(model):
    rng = np.random.default_rng(0)
    eng = _engine(model, 7, 2, 33, 5)
    ent, rel = _tables(model, 33, 5, 7, rng)
    eng.set_embeddings(ent, rel)
    assert (_dense(eng, eng.ent) == ent).all() and (_dense(eng, eng.rel) == rel).all()
    e2, r2 = eng.get_embeddings()
    assert (e2.cpu().numpy() == ent).all() and (r2.cpu().numpy() == rel).all()
    pad = eng.ent.cpu().numpy()[:, 7:8]
    assert (pad == 0).all()


def test_reference_scoring_kats_on_gpu(kats):
    """The reference's own golden vectors, through kge_score_triples."""
    from oracle import c_oracle  # checker only
    for c in kats["scoring"]:
        if c["form"] != "triple":
            continue
        e_s, e_p, e_o = (np.array(c[x], np.float32) for x in ("e_s", "e_p", "e_o"))
        n = len(e_s)
        R = c["max_rel_size"] or n
        rel = np.zeros((max(R, n), e_p.shape[1]), np.float32)
        rel[:n] = e_p
        eng = _engine(c["model"], c["k"], 1, 2 * n, max(R, n))
        # RotatE's phase normalisation uses n_rel == max_rel_size of the KAT
        assert eng.n_rel == (c["max_rel_size"] or n)
        eng.set_embeddings(np.concatenate([e_s, e_o]), rel[:eng.n_rel])
        t = np.stack([np.arange(n), np.arange(n), n + np.arange(n)], 1).astype(np.int32)
        got = np.around(eng.score(_dev(t)).cpu().numpy(), c["round_decimals"])
        assert (got == np.array(c["expected"], np.float32)).all(), (c["source"], got)
        eng.close()


def _score_tables(model, E, R, k, kind, rng):
    """Glorot tables; 'scaled': every row times 2^e, e uniform in [-20, 20] (RotatE: entity rows only, its phases stay
    in range), so that small scores sit beside large ones; 'subnormal': a tenth of the rows (RotatE: entity rows) with
    subnormal entries in half their columns; 'nonfinite': +inf, -inf and NaN in a few entity rows (and one relation row
    but RotatE's), every finite value far from overflow."""
    ent, rel = _tables(model, E, R, k, rng)
    K = ent.shape[1]
    tabs = ((ent, E), (rel, R)) if model != "RotatE" else ((ent, E),)
    if kind == "scaled":
        for tab, rows in tabs:
            tab *= (2.0 ** rng.integers(-20, 21, rows))[:, None].astype(np.float32)
    elif kind == "subnormal":
        for tab, rows in tabs:
            for r in rng.choice(rows, max(1, rows // 10), replace=False):
                cols = rng.random(K) < 0.5
                tab[r, cols] = (rng.uniform(-1, 1, int(cols.sum())) * 2.0 ** -126).astype(np.float32)
    elif kind == "nonfinite":
        for v, r in zip((np.inf, -np.inf, np.nan) * 4, rng.choice(E, 12, replace=False)):
            ent[r, rng.integers(0, K)] = v
        if model != "RotatE":
            rel[1, rng.integers(0, K)] = np.inf
    return ent, rel


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("k", [1, 5, 31, 32, 33, 50, 100, 130, 200, 1000])
def test_score_triples_vs_oracle(model, k):
    """kge_score_triples (the predict path) against the float64 oracle, every score within exact_oracle.PredictBound:
    n = 1, 7 and 20,000 triples (more than the grid's 64 warps per SM, so the grid-stride loop wraps) on Glorot,
    row-scaled and subnormal tables, and RotatE with max_rel_size != n_rel; non-finite entries give NaN / +inf / -inf
    exactly where the oracle does.  Sensitivity: the check rejects the kernel's scores against an oracle whose one entity
    element is multiplied by 1 + 2^-10 (an element made dominant in its row, 32 times the Glorot limit, so that it
    carries a few percent of its triple's |score|_abs even at k = 1,000)."""
    import exact_oracle as xo
    E, R = 3000, 11
    rng = np.random.default_rng(zlib.crc32(repr((model, k)).encode()))
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    big = max(20000, 64 * sm + 1000)
    runs = [("glorot", None), ("scaled", None), ("subnormal", None), ("nonfinite", None)]
    if model == "RotatE":
        runs.append(("glorot", 3 * R + 2))
    ratios = {}
    for kind, mrs in runs:
        ent, rel = _score_tables(model, E, R, k, kind, rng)
        t_big = _triples(E, R, big, rng)
        if kind == "glorot" and mrs is None:  # the sensitivity probe: triple 0's subject row, its dominant element
            e = int(t_big[0, 0])
            x = torch.as_tensor(ent, dtype=torch.float64)
            s = x[t_big[:1, 0]].clone().requires_grad_(True)
            xo.scores(model, s, torch.as_tensor(rel, dtype=torch.float64)[t_big[:1, 1]], x[t_big[:1, 2]], R,
                      rot_table=True).sum().backward()
            j = int((s.grad[0] * s.detach()[0]).abs().argmax())
            ent[e, j] = np.float32(32 * np.sqrt(6.0 / (E + ent.shape[1])) * (1 if ent[e, j] >= 0 else -1))
        eng = _engine(model, k, 2, E, R, max_rel_size=mrs)
        eng.set_embeddings(ent, rel)
        for n in (1, 7, big):
            t = t_big[:n]
            got = eng.score(_dev(t)).cpu().numpy()
            bound = xo.PredictBound(model, ent, rel, t, max_rel_size=mrs, device="cuda")
            where = "%s k=%d %s max_rel_size=%s n=%d" % (model, k, kind, mrs, n)
            if kind == "nonfinite":
                ok, ratio, i = bound.check(got)
                assert ok, (where, i, t[i].tolist(), float(got[i]), float(bound.want[i]))
                assert n < big or not np.isfinite(got).all(), where
            else:
                assert np.isfinite(got).all(), where
                ratio = bound.assert_within(got, where)
            ratios["%s%s n=%d" % (kind, "" if mrs is None else " mrs=%d" % mrs, n)] = round(ratio, 4)
        if kind == "glorot" and mrs is None:  # sensitivity, on the n = 20,000 run
            ent2 = ent.copy()
            ent2[e, j] *= np.float32(1 + 2.0 ** -10)
            rows = np.nonzero((t[:, 0] == e) | (t[:, 2] == e))[0]
            want2 = xo.PredictBound(model, ent2, rel, t[rows], device="cuda").want
            assert not bound.check(got[rows], want=want2, rows=rows)[0], "%s k=%d: the check accepts a perturbed " \
                "entity element" % (model, k)
        eng.close()
    print("\n%s k=%d: worst error / bound %s" % (model, k, ratios))


# ---------------------------------------------------------------------------
def _ref(model, k, ent, rel, eta, loss, lp, **kw):
    from oracle import ref_step
    p = dict(lp)
    return ref_step.RefStep(model, ent.shape[1], ent, rel, eta, loss=loss,
                            loss_params={k_: v for k_, v in p.items()}, **kw)


def _corruption_tensor(t, neg_ent, neg_keep, eta):
    from oracle import c_oracle
    return c_oracle.corrupt(t, eta, neg_keep, neg_ent)


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("loss", LOSSES)
@pytest.mark.parametrize("reduction", ["sum", "mean"])
def test_forward_backward_vs_oracle(model, loss, reduction):
    rng = np.random.default_rng(hash((model, loss, reduction)) % 2**32)
    E, R, k, eta, B = 64, 5, 12, 5, 97
    ent, rel = _tables(model, E, R, k, rng, scale=0.6)
    t = _triples(E, R, B, rng)
    neg_ent, neg_keep = _negatives(E, B, eta, rng)
    lp = {"reduction": reduction}
    if loss in ("pairwise", "absolute_margin"):
        lp["margin"] = 0.5
    if loss == "self_adversarial":
        lp.update(margin=2.0, alpha=0.7)
    eng = _engine(model, k, eta, E, R, loss=loss, loss_params=lp)
    eng.set_embeddings(ent, rel)
    sp = torch.empty(B, device="cuda")
    sn = torch.empty(B * eta, device="cuda")
    eng.forward_backward(_dev(t), (_dev(neg_ent), _dev(neg_keep)), scores_pos=sp, scores_neg=sn)
    rs = _ref(model, k, ent, rel, eta, loss, lp)
    rl, rsp, rsn, g_ent, g_rel = rs.loss_and_grads(t, _corruption_tensor(t, neg_ent, neg_keep, eta))
    assert np.allclose(sp.cpu().numpy(), rsp.numpy(), rtol=RTOL, atol=1e-5)
    assert np.allclose(sn.cpu().numpy(), rsn.numpy(), rtol=RTOL, atol=1e-5)
    assert abs(eng.read_loss() - float(rl)) <= RTOL * abs(float(rl)) + 1e-5
    assert _close(_dense(eng, eng.g_ent), g_ent.numpy()), np.abs(_dense(eng, eng.g_ent) - g_ent.numpy()).max()
    assert _close(_dense(eng, eng.g_rel), g_rel.numpy()), np.abs(_dense(eng, eng.g_rel) - g_rel.numpy()).max()
    eng.close()


@pytest.mark.parametrize("model,k,eta,B", [("ComplEx", 200, 10, 300), ("DistMult", 400, 20, 200),
                                           ("RotatE", 200, 30, 150), ("TransE", 50, 2, 1000),
                                           ("HolE", 130, 7, 123)])
def test_forward_backward_baseline_shapes(model, k, eta, B):
    """BASELINE.json config shapes (k, eta) on a reduced KG."""
    rng = np.random.default_rng(7)
    E, R = 500, 11
    loss = {"ComplEx": "self_adversarial", "RotatE": "self_adversarial"}.get(model, "pairwise")
    ent, rel = _tables(model, E, R, k, rng)
    t = _triples(E, R, B, rng)
    neg_ent, neg_keep = _negatives(E, B, eta, rng)
    eng = _engine(model, k, eta, E, R, loss=loss)
    eng.set_embeddings(ent, rel)
    eng.forward_backward(_dev(t), (_dev(neg_ent), _dev(neg_keep)))
    rs = _ref(model, k, ent, rel, eta, loss, {})
    rl, _, _, g_ent, g_rel = rs.loss_and_grads(t, _corruption_tensor(t, neg_ent, neg_keep, eta))
    assert abs(eng.read_loss() - float(rl)) <= RTOL * abs(float(rl))
    assert _close(_dense(eng, eng.g_ent), g_ent.numpy())
    assert _close(_dense(eng, eng.g_rel), g_rel.numpy())
    eng.close()


@pytest.mark.parametrize("model,loss,eta,B", [("ComplEx", "self_adversarial", 40, 37), ("TransE", "multiclass_nll", 70, 9),
                                              ("RotatE", "self_adversarial", 33, 21), ("DistMult", "nll", 1, 1),
                                              ("HolE", "pairwise", 1, 300)])
def test_edge_shapes_eta_over_32_and_tiny_batches(model, loss, eta, B):
    """eta > 32 (several corruptions per lane in the loss, more than one ballot word), eta = 1, B = 1."""
    rng = np.random.default_rng(47)
    E, R, k = 90, 3, 10
    ent, rel = _tables(model, E, R, k, rng, scale=0.4)
    t = _triples(E, R, B, rng)
    neg_ent, neg_keep = _negatives(E, B, eta, rng)
    eng = _engine(model, k, eta, E, R, loss=loss)
    eng.set_embeddings(ent, rel)
    sn = torch.empty(B * eta, device="cuda")
    sp = torch.empty(B, device="cuda")
    eng.forward_backward(_dev(t), (_dev(neg_ent), _dev(neg_keep)), scores_pos=sp, scores_neg=sn)
    rs = _ref(model, k, ent, rel, eta, loss, {})
    rl, rsp, rsn, g_ent, g_rel = rs.loss_and_grads(t, _corruption_tensor(t, neg_ent, neg_keep, eta))
    assert np.allclose(sn.cpu().numpy(), rsn.numpy(), rtol=RTOL, atol=1e-5)
    assert abs(eng.read_loss() - float(rl)) <= RTOL * abs(float(rl)) + 1e-5
    assert _close(_dense(eng, eng.g_ent), g_ent.numpy()) and _close(_dense(eng, eng.g_rel), g_rel.numpy())
    # an empty batch is a no-op
    eng.g_ent.zero_(); eng.g_rel.zero_()
    eng.forward_backward(torch.empty((0, 3), dtype=torch.int32, device="cuda"), None)
    assert eng.read_loss() == 0 and (eng.g_ent == 0).all()
    assert eng.score(torch.empty((0, 3), dtype=torch.int32, device="cuda")).numel() == 0
    assert eng.rank(torch.empty((0, 3), dtype=torch.int32, device="cuda"), "s").numel() == 0
    eng.close()


@pytest.mark.parametrize("model,k", [("TransE", 600), ("DistMult", 1100), ("ComplEx", 520), ("HolE", 1000), ("RotatE", 700)])
@pytest.mark.parametrize("group", [0, 3])
def test_wide_rows_column_windows(model, k, group):
    """half-rows wider than 512 floats are processed in column windows (cfg5 has k=1000), with and
    without negative groups; compared with the oracle."""
    rng = np.random.default_rng(41)
    E, R, eta, B = 60, 4, 7, 41
    loss = "self_adversarial" if model in ("ComplEx", "RotatE") else "nll"
    ent, rel = _tables(model, E, R, k, rng, scale=0.05)
    t = _triples(E, R, B, rng)
    neg_ent, neg_keep = _negatives(E, B, eta, rng)
    eng = _engine(model, k, eta, E, R, loss=loss, neg_group=group)
    eng.set_embeddings(ent, rel)
    sp = torch.empty(B, device="cuda")
    sn = torch.empty(B * eta, device="cuda")
    eng.forward_backward(_dev(t), (_dev(neg_ent), _dev(neg_keep)), scores_pos=sp, scores_neg=sn)
    rs = _ref(model, k, ent, rel, eta, loss, {})
    rl, rsp, rsn, g_ent, g_rel = rs.loss_and_grads(t, _corruption_tensor(t, neg_ent, neg_keep, eta))
    assert np.allclose(sp.cpu().numpy(), rsp.numpy(), rtol=RTOL, atol=1e-5)
    assert np.allclose(sn.cpu().numpy(), rsn.numpy(), rtol=RTOL, atol=1e-5)
    assert abs(eng.read_loss() - float(rl)) <= RTOL * abs(float(rl)) + 1e-5
    assert _close(_dense(eng, eng.g_ent), g_ent.numpy()) and _close(_dense(eng, eng.g_rel), g_rel.numpy())
    eng.close()


@pytest.mark.parametrize("model", ["ComplEx", "TransE", "RotatE"])
@pytest.mark.parametrize("group", [1, 3])
def test_negative_groups_match_resident(model, group):
    """eta negatives processed in groups of G (two-pass path) == all-resident path."""
    rng = np.random.default_rng(11)
    E, R, k, eta, B = 80, 4, 20, 7, 64
    ent, rel = _tables(model, E, R, k, rng, scale=0.5)
    t = _triples(E, R, B, rng)
    neg = _negatives(E, B, eta, rng)
    outs = []
    for g in (0, group):
        eng = _engine(model, k, eta, E, R, loss="self_adversarial", neg_group=g)
        eng.set_embeddings(ent, rel)
        eng.forward_backward(_dev(t), (_dev(neg[0]), _dev(neg[1])))
        outs.append((_dense(eng, eng.g_ent), _dense(eng, eng.g_rel), eng.read_loss()))
        eng.close()
    assert _close(outs[1][0], outs[0][0]) and _close(outs[1][1], outs[0][1])
    assert abs(outs[1][2] - outs[0][2]) <= RTOL * abs(outs[0][2])


@pytest.mark.parametrize("model,k,group", [("ComplEx", 20, 3), ("RotatE", 24, 2), ("TransE", 600, 3), ("ComplEx", 520, 0),
                                           ("DistMult", 1100, 1)])
def test_row_stash_matches_second_gather(model, k, group):
    """kge_set_row_stash: the gradient pass re-reads the replaced rows from the stash the score pass filled; same
    gradients as gathering them twice, and the stash holds exactly the gathered table rows."""
    rng = np.random.default_rng(23)
    E, R, eta, B = 90, 4, 7, 70
    ent, rel = _tables(model, E, R, k, rng, scale=0.3 if k < 100 else 0.05)
    t = _triples(E, R, B, rng)
    neg = _negatives(E, B, eta, rng)
    outs = []
    for stash in (False, True):
        eng = _engine(model, k, eta, E, R, loss="self_adversarial", neg_group=group)
        eng.set_embeddings(ent, rel)
        if stash:
            st = eng.ensure_row_stash(B)
            assert st is not None, "expected a non-resident geometry"
            st.fill_(float("nan"))
        eng.forward_backward(_dev(t), (_dev(neg[0]), _dev(neg[1])))
        outs.append((_dense(eng, eng.g_ent), _dense(eng, eng.g_rel), eng.read_loss()))
        if stash:
            torch.cuda.synchronize()
            # stash row i*eta+t holds slot t of positive i: the corruptions that replaced the subject (keep_subj == 0)
            # in draw order, then those that replaced the object (the kernel sorts by side as it draws)
            ids = neg[0].reshape(eta, B).T
            keep = neg[1].reshape(eta, B).T
            order = np.argsort(keep, axis=1, kind="stable")
            want = eng.ent[_dev(np.take_along_axis(ids, order, axis=1).reshape(-1)).long()]
            assert torch.equal(st[:B * eta], want)
        eng.close()
    assert _close(outs[1][0], outs[0][0]) and _close(outs[1][1], outs[0][1])
    assert abs(outs[1][2] - outs[0][2]) <= RTOL * abs(outs[0][2])


def test_philox_corruptions_structure_and_parity():
    """In-kernel Philox negatives: structure of A3 + the fused kernel really uses that stream."""
    rng = np.random.default_rng(13)
    E, R, k, eta, B = 1000, 10, 16, 4, 500
    ent, rel = _tables("DistMult", E, R, k, rng, scale=0.5)
    t = _triples(E, R, B, rng)
    eng = _engine("DistMult", k, eta, E, R, loss="nll")
    eng.set_embeddings(ent, rel)
    corr = eng.generate_corruptions(_dev(t), seed=5, step=3).cpu().numpy()
    assert corr.shape == (B * eta, 3)
    tiled = np.tile(t, (eta, 1))
    assert (corr[:, 1] == tiled[:, 1]).all()  # relation kept
    s_same, o_same = corr[:, 0] == tiled[:, 0], corr[:, 2] == tiled[:, 2]
    assert (s_same | o_same).all()  # at most one side replaced
    assert corr.min() >= 0 and corr.max() < E
    frac_obj = (s_same & ~o_same).mean()
    assert 0.4 < frac_obj < 0.6  # keep_subj ~ Bernoulli(1/2)
    repl = np.where(~s_same, corr[:, 0], corr[:, 2])
    assert abs(repl.mean() - (E - 1) / 2) < 0.05 * E  # uniform replacement ids
    corr2 = eng.generate_corruptions(_dev(t), seed=5, step=4).cpu().numpy()
    assert (corr2 != corr).any()  # the stream advances with the step
    # the device draw is the published Philox4x32-10 stream: bit-identical to the library's CPU replay and to the
    # oracle's independent statement of it (oracle/philox.py, pinned by the Random123 known answers)
    from ampligraph_b200 import _lib
    from oracle import philox
    assert (corr == _lib.host_corruptions(t, eta, E, seed=5, step=3)).all()
    assert (corr[:64] == philox.corruption_stream(t, eta, E, 5, 3)[:64]).all()
    # gradients of the Philox path == oracle fed with the materialised corruptions
    eng.forward_backward(_dev(t), None, seed=5, step=3)
    rs = _ref("DistMult", k, ent, rel, eta, "nll", {})
    rl, _, _, g_ent, g_rel = rs.loss_and_grads(t, corr)
    assert abs(eng.read_loss() - float(rl)) <= RTOL * abs(float(rl))
    assert _close(_dense(eng, eng.g_ent), g_ent.numpy()) and _close(_dense(eng, eng.g_rel), g_rel.numpy())
    eng.close()


@pytest.mark.parametrize("opt,params", [("adam", {}), ("adam", {"learning_rate": 0.01, "beta_1": 0.8}),
                                        ("sgd", {"learning_rate": 0.05}), ("sgd", {"learning_rate": 0.05, "momentum": 0.9}),
                                        ("adagrad", {"learning_rate": 0.1})])
@pytest.mark.parametrize("reg", [None, {"p": 2, "lambda": 1e-3}, {"p": 3, "lambda": 1e-2}])
def test_train_steps_vs_oracle(opt, params, reg):
    """several full steps (fwd+bwd+optimizer+regulariser) track the op-for-op restatement."""
    rng = np.random.default_rng(17)
    model, E, R, k, eta, B = "ComplEx", 50, 4, 10, 3, 40
    ent, rel = _tables(model, E, R, k, rng, scale=0.5)
    eng = _engine(model, k, eta, E, R, loss="multiclass_nll", optimizer=opt, optimizer_params=params, regularizer=reg)
    eng.set_embeddings(ent, rel)
    rs = _ref(model, k, ent, rel, eta, "multiclass_nll", {}, optimizer=opt, optimizer_params=dict(params),
              regularizer=({"p": reg["p"], "lam": reg["lambda"]} if reg else None))
    for step in range(5):
        t = _triples(E, R, B, rng)
        neg_ent, neg_keep = _negatives(E, B, eta, rng)
        eng.train_step(_dev(t), (_dev(neg_ent), _dev(neg_keep)))
        ref_loss = rs.train_step(t, _corruption_tensor(t, neg_ent, neg_keep, eta))
        got_loss = eng.read_loss()
        assert abs(got_loss - ref_loss) <= 2e-4 * abs(ref_loss), (step, got_loss, ref_loss)
        assert (eng.g_ent == 0).all() and (eng.g_rel == 0).all()  # accumulators cleared for the next step
    assert _close(_dense(eng, eng.ent), rs.ent.detach().numpy(), rtol=5e-4)
    assert _close(_dense(eng, eng.rel), rs.rel.detach().numpy(), rtol=5e-4)
    eng.close()


LAZY_OPTS = ["lazy_adam", "lazy_adagrad", "lazy_sgd"]
# DistMult runs the resident trilinear kernel, RotatE the RotatE kernel, ComplEx with neg_group = 3 the general kernel: each
# stamps the rows it touches itself (DistMult keeps its original test ids)
LAZY_CASES = ([pytest.param(opt, "DistMult", 0, id=opt) for opt in LAZY_OPTS] +
              [pytest.param(opt, m, g, id="%s-%s" % (m, opt)) for m, g in (("RotatE", 0), ("ComplEx", 3)) for opt in LAZY_OPTS])


@pytest.mark.parametrize("opt,model,neg_group", LAZY_CASES)
def test_lazy_optimizer_matches_restatement(opt, model, neg_group):
    """opt-in lazy optimizer (rows touched by the step only) vs the oracle's lazy restatement; untouched
    rows must not move at all."""
    rng = np.random.default_rng(43)
    E, R, k, eta, B = 400, 6, 12, 3, 25   # few positives: most rows stay untouched
    ent, rel = _tables(model, E, R, k, rng, scale=0.5)
    eng = _engine(model, k, eta, E, R, loss="nll", optimizer=opt, optimizer_params={"learning_rate": 0.01}, neg_group=neg_group)
    eng.set_embeddings(ent, rel)
    rs = _ref(model, k, ent, rel, eta, "nll", {}, optimizer=opt, optimizer_params={"learning_rate": 0.01})
    touched = np.zeros(E, bool)
    for step in range(4):
        t = _triples(E, R, B, rng)
        neg_ent, neg_keep = _negatives(E, B, eta, rng)
        eng.train_step(_dev(t), (_dev(neg_ent), _dev(neg_keep)), step=step)
        rs.train_step(t, _corruption_tensor(t, neg_ent, neg_keep, eta))
        touched[t[:, 0]] = touched[t[:, 2]] = touched[neg_ent] = True
        assert (eng.g_ent == 0).all()
    got = _dense(eng, eng.ent)
    assert _close(got, rs.ent.detach().numpy(), rtol=5e-4) and _close(_dense(eng, eng.rel), rs.rel.detach().numpy(), rtol=5e-4)
    assert (~touched).sum() > 50 and (got[~touched] == ent[~touched]).all()
    eng.close()


def test_external_loss_two_phase():
    """LossFunctionWrapper path (loss_functions.py:657): scores out, dL/dscore back in."""
    rng = np.random.default_rng(19)
    model, E, R, k, eta, B = "HolE", 40, 3, 9, 4, 33
    ent, rel = _tables(model, E, R, k, rng, scale=0.5)
    t = _triples(E, R, B, rng)
    neg_ent, neg_keep = _negatives(E, B, eta, rng)
    eng = _engine(model, k, eta, E, R)
    eng.set_embeddings(ent, rel)
    from ampligraph_b200 import _lib
    sp = torch.empty(B, device="cuda")
    sn = torch.empty(B * eta, device="cuda")
    negs = (_dev(neg_ent), _dev(neg_keep))
    eng.forward_backward(_dev(t), negs, mode=_lib.STEP_FORWARD_ONLY, scores_pos=sp, scores_neg=sn)
    assert (eng.g_ent == 0).all()

    def user_loss(scores_pos, scores_neg):  # the docstring example of the reference (:660-668)
        neg_exp, pos_exp = torch.exp(scores_neg), torch.exp(scores_pos)
        return -torch.log(pos_exp / (neg_exp.sum(0) + pos_exp))

    spg, sng = sp.clone().requires_grad_(True), sn.clone().requires_grad_(True)
    user_loss(spg, sng.reshape(eta, -1)).sum().backward()
    eng.forward_backward(_dev(t), negs, mode=_lib.STEP_BACKWARD_EXT, dpos=spg.grad.contiguous(), dneg=sng.grad.contiguous())
    from oracle import ref_step
    rs = _ref(model, k, ent, rel, eta, "pairwise", {})
    rsp, rsn = rs.forward(t, _corruption_tensor(t, neg_ent, neg_keep, eta))
    user_loss(rsp, rsn.reshape(eta, -1)).sum().backward()
    assert _close(_dense(eng, eng.g_ent), rs.ent.grad.numpy()) and _close(_dense(eng, eng.g_rel), rs.rel.grad.numpy())
    eng.close()


def _zipf_triples(E, R, n, rng):
    """s,o ~ truncated Zipf(1.0) over a random permutation: hot entities collide in the red.v4 scatter like real data."""
    w = 1.0 / np.arange(1, E + 1)
    cdf = np.cumsum(w / w.sum())
    perm = rng.permutation(E)
    s, o = perm[np.searchsorted(cdf, rng.random(n))], perm[np.searchsorted(cdf, rng.random(n))]
    return np.stack([s, rng.integers(0, R, n), o], 1).astype(np.int32)


@pytest.mark.parametrize("name,model,k,eta,E,R,B,loss", [
    # BASELINE configs[1] and [2] at their FULL stated size (entities, batch), Zipf-distributed triples
    ("cfg2", "ComplEx", 200, 10, 14505, 237, 27212, "self_adversarial"),
    ("cfg3", "DistMult", 400, 20, 40943, 11, 8684, "pairwise"),
    # configs[3] and [4]: exact (k, eta) and a table that does not fit the H100's 50 MB L2 (197 MB / 800 MB); the batch is
    # bounded so that the CPU oracle (which materialises [B*eta, K] tensors) finishes in seconds
    ("cfg4", "RotatE", 200, 30, 123182, 37, 2048, "self_adversarial"),
    ("cfg5", "ComplEx", 1000, 50, 100000, 1000, 512, "self_adversarial"),
])
def test_full_size_forward_backward_vs_oracle(name, model, k, eta, E, R, B, loss):
    """The fused kernel against the INDEPENDENT oracle (oracle/ref_step.py: 6 gathers, broadcast scoring, autograd) at
    BASELINE sizes: loss and both gradient tables within 1e-4 (VERDICT r1 #2; replaces the self-referential
    gradient-linearity check).  Zipf-heavy collisions in the red.v4 scatter, column windows (cfg5) and negative
    groups (cfg4, cfg5) are all exercised against an answer the kernel did not produce."""
    rng = np.random.default_rng(101)
    ent, rel = _tables(model, E, R, k, rng)
    t = _zipf_triples(E, R, B, rng)
    neg_ent, neg_keep = _negatives(E, B, eta, rng)
    lp = {"margin": 3.0, "alpha": 0.5} if loss == "self_adversarial" else {"margin": 1.0}
    eng = _engine(model, k, eta, E, R, loss=loss, loss_params=lp)
    eng.set_embeddings(ent, rel)
    eng.forward_backward(_dev(t), (_dev(neg_ent), _dev(neg_keep)))
    got_loss = eng.read_loss()
    g_e, g_r = _dense(eng, eng.g_ent), _dense(eng, eng.g_rel)
    pads_zero = bool((eng.g_ent[:, eng.k:eng.kp] == 0).all())
    resident = eng.lib.kge_rows_resident(eng.h)
    eng.close()
    assert resident == (1 if name == "cfg2" else 0)  # cfg3 (23 rows of 1600 B per positive), cfg4, cfg5: grouped / windowed path
    rs = _ref(model, k, ent, rel, eta, loss, lp)
    rl, _, _, r_e, r_r = rs.loss_and_grads(t, _corruption_tensor(t, neg_ent, neg_keep, eta))
    assert abs(got_loss - float(rl)) <= RTOL * abs(float(rl)), (got_loss, float(rl))
    assert _close(g_e, r_e.numpy()), np.abs(g_e - r_e.numpy()).max() / np.abs(r_e.numpy()).max()
    assert _close(g_r, r_r.numpy()), np.abs(g_r - r_r.numpy()).max() / np.abs(r_r.numpy()).max()
    assert pads_zero


def test_gradient_linearity_full_size():
    """cfg2 at full size: grads(A u B) == grads(A) + grads(B), loss additive (a size-independent property, kept beside
    the oracle comparison above)."""
    rng = np.random.default_rng(23)
    model, E, R, k, eta, B = "ComplEx", 14505, 237, 200, 10, 27212
    eng = _engine(model, k, eta, E, R, loss="self_adversarial")
    eng.init_glorot_uniform(seed=1)
    t = _dev(_triples(E, R, B, rng))
    neg_ent, neg_keep = _negatives(E, B, eta, rng)
    ne, nk = _dev(neg_ent), _dev(neg_keep)
    eng.forward_backward(t, (ne, nk))
    g_all, gr_all, loss_all = eng.g_ent.clone(), eng.g_rel.clone(), eng.read_loss()
    eng.g_ent.zero_(); eng.g_rel.zero_()
    h = B // 2
    idx = torch.arange(B, device="cuda")
    for sel in (idx[:h], idx[h:]):
        rows = (torch.arange(eta, device="cuda")[:, None] * B + sel[None, :]).reshape(-1)
        eng.forward_backward(t[sel].contiguous(), (ne[rows].contiguous(), nk[rows].contiguous()))
    loss_parts = eng.read_loss()
    assert abs(loss_parts - loss_all) <= 1e-5 * abs(loss_all)
    scale = g_all.abs().max().item()
    assert (eng.g_ent - g_all).abs().max().item() <= 1e-4 * scale
    assert (eng.g_rel - gr_all).abs().max().item() <= 1e-4 * gr_all.abs().max().item()
    eng.close()


def test_initializers_bound_mean_std():
    """The reference pins its initialisers by mean/std only (tests/ampligraph/latent_features/test_initializers.py:40-49:
    RandomNormal(mean=0.5, stddev=0.05) -> |mean-0.5|, |std-0.05| small).  Same check through kge_init_table /
    kge_init_glorot_uniform, plus the Glorot bound sqrt(6/(rows+K)) (EmbeddingLookupLayer.py:194-201), truncation at
    2 stddev, zero pad columns, and seed dependence."""
    E, R, k = 20000, 50, 37  # k not a multiple of 4: pad columns exist
    eng = _engine("ComplEx", k, 1, E, R)
    K = eng.internal_k
    eng.init_glorot_uniform(seed=3)
    ent = _dense(eng, eng.ent)
    lim = np.sqrt(6.0 / (E + K))
    assert np.abs(ent).max() <= lim and np.abs(ent).max() > 0.999 * lim
    assert abs(ent.mean()) < 0.01 * lim and abs(ent.std() - lim / np.sqrt(3)) < 0.01 * lim
    assert (eng.ent[:, k:eng.kp] == 0).all() and (eng.ent[:, eng.kp + k:] == 0).all()
    rel = _dense(eng, eng.rel)
    assert np.abs(rel).max() <= np.sqrt(6.0 / (R + K))
    eng.init_glorot_uniform(seed=4)
    assert (np.abs(_dense(eng, eng.ent) - ent) > 0).mean() > 0.99  # another seed, another table
    eng.init_table("ent", "normal", 0.5, 0.05, seed=1)
    x = _dense(eng, eng.ent)
    assert abs(x.mean() - 0.5) < 1e-3 and abs(x.std() - 0.05) < 1e-3  # the reference's own test, 1e-1 there
    assert (eng.ent[:, k:eng.kp] == 0).all()
    eng.init_table("ent", "truncated_normal", 0.0, 1.0, seed=1)
    x = _dense(eng, eng.ent)
    assert np.abs(x).max() <= 2.0 and abs(x.std() - 0.87962566) < 5e-3 and abs(x.mean()) < 5e-3
    eng.init_table("rel", "uniform", -0.25, 0.75, seed=2)
    x = _dense(eng, eng.rel)
    assert x.min() >= -0.25 and x.max() < 0.75 and abs(x.mean() - 0.25) < 0.02
    eng.init_table("rel", "constant", 1.0)
    assert (_dense(eng, eng.rel) == 1.0).all()
    eng.close()


def test_regulariser_pair_and_l1_l2():
    """A [entities, relations] pair of regularisers (EmbeddingLookupLayer.py:131-155) and Keras' l1_l2 (two LP terms):
    one optimizer step against the oracle, loss included."""
    rng = np.random.default_rng(59)
    model, E, R, k, eta, B = "DistMult", 60, 5, 8, 2, 30
    ent, rel = _tables(model, E, R, k, rng, scale=0.5)
    regs = [{"p": 1, "lambda": 1e-2, "p2": 2, "lambda2": 3e-2}, {"p": 3, "lambda": 2e-2}]
    eng = _engine(model, k, eta, E, R, loss="nll", optimizer="sgd", optimizer_params={"learning_rate": 0.1}, regularizer=regs)
    eng.set_embeddings(ent, rel)
    t = _triples(E, R, B, rng)
    neg_ent, neg_keep = _negatives(E, B, eta, rng)
    eng.train_step(_dev(t), (_dev(neg_ent), _dev(neg_keep)))
    rs = _ref(model, k, ent, rel, eta, "nll", {})
    rl, _, _, g_e, g_r = rs.loss_and_grads(t, _corruption_tensor(t, neg_ent, neg_keep, eta))
    g_e, g_r = g_e.numpy().astype(np.float64), g_r.numpy().astype(np.float64)
    g_e += 1e-2 * np.sign(ent) + 3e-2 * 2 * ent
    g_r += 2e-2 * 3 * np.abs(rel) ** 2 * np.sign(rel)
    want_loss = float(rl) + 1e-2 * np.abs(ent).sum() + 3e-2 * (ent.astype(np.float64) ** 2).sum() + 2e-2 * (np.abs(rel).astype(np.float64) ** 3).sum()
    assert abs(eng.read_loss() - want_loss) <= 2e-4 * abs(want_loss)
    assert _close(_dense(eng, eng.ent), ent - 0.1 * g_e, rtol=2e-4) and _close(_dense(eng, eng.rel), rel - 0.1 * g_r, rtol=2e-4)
    eng.close()


@pytest.mark.parametrize("model,k,eta", [("ComplEx", 200, 10), ("HolE", 50, 7), ("DistMult", 200, 32), ("ComplEx", 30, 1), ("DistMult", 7, 3),
                                         ("DistMult", 400, 20), ("DistMult", 509, 9),  # NIT = 4 rows (cfg3's shape)
                                         # kge_train_rot_kernel: cfg4's shape (4 groups of 8), everything resident, eta > 32 (two
                                         # ballot rounds), 5 groups with a short last one, NIT = 1 in groups
                                         ("RotatE", 200, 30), ("RotatE", 50, 7), ("RotatE", 20, 40), ("RotatE", 256, 33), ("RotatE", 100, 90)])
def test_resident_fast_path_equals_general_kernel(model, k, eta, monkeypatch):
    """kge_train_res_kernel / kge_train_rot_kernel (the fast paths) against kge_train_kernel forced by KGE_B200_TRAIN_KERNEL=general:
    identical arithmetic per score, so scores are bit-equal; gradients agree to atomic-order noise; both match the oracle
    elsewhere (test_forward_backward_vs_oracle runs through the fast path by default)."""
    rng = np.random.default_rng(71)
    E, R, B = 900, 9, 777
    ent, rel = _tables(model, E, R, k, rng, scale=0.3)
    t = _triples(E, R, B, rng)
    hot = rng.random(B)
    t[hot < 0.2, 0] = 5; t[(hot > 0.15) & (hot < 0.4), 2] = 5; t[hot > 0.85, 0] = 17; t[(hot > 0.6) & (hot < 0.7), 2] = 17  # skewed graph
    neg_ent, neg_keep = _negatives(E, B, eta, rng)
    out = {}
    for which in ("fast", "fast_hot", "general"):
        if which == "general":
            monkeypatch.setenv("KGE_B200_TRAIN_KERNEL", "general")
        else:
            monkeypatch.delenv("KGE_B200_TRAIN_KERNEL", raising=False)
        eng = _engine(model, k, eta, E, R, loss="self_adversarial")
        # (the general kernel processes cfg3's shape in groups of corruptions; the fast path keeps all of them resident on 6 warps)
        assert eng.lib.kge_rows_resident(eng.h) or (model, k, eta) == ("DistMult", 400, 20) or model == "RotatE"
        if which == "fast_hot":  # kge_set_hot_entities: entities 5 and 17 are summed per warp and scattered once
            eng.set_hot_entities(triples=t)
            assert sorted(eng.hot_entities) == [5, 17]
        eng.set_embeddings(ent, rel)
        sp = torch.empty(B, device="cuda"); sn = torch.empty(eta * B, device="cuda")
        eng.forward_backward(_dev(t), (_dev(neg_ent), _dev(neg_keep)), scores_pos=sp, scores_neg=sn)
        torch.cuda.synchronize()
        out[which] = (sp.cpu().numpy(), sn.cpu().numpy(), eng.g_ent.cpu().numpy().copy(), eng.g_rel.cpu().numpy().copy(), eng.read_loss())
        eng.close()
    g = out["general"]
    for which in ("fast", "fast_hot"):
        f = out[which]
        assert (f[0] == g[0]).all() and (f[1] == g[1]).all(), which
        assert _close(f[2], g[2], rtol=2e-5) and _close(f[3], g[3], rtol=2e-5), which
        assert abs(f[4] - g[4]) <= 1e-6 * abs(g[4]), which


@pytest.mark.parametrize("model,k,E,B", [("ComplEx", 40, 700, 9000), ("DistMult", 400, 300, 4000), ("RotatE", 200, 400, 3000)])
def test_dynamic_assignment_of_positives_equals_static_stride(model, k, E, B, monkeypatch):
    """KGE_B200_TRAIN_SCHED=dynamic (positives drawn from a self-resetting counter, kge_train_common.cuh) against the static
    stride: which warp processes a positive does not change its arithmetic, so scores are bit-equal and the gradients agree to
    atomic-order noise; three consecutive launches on one handle check that the counter resets itself."""
    rng = np.random.default_rng(83)
    R, eta = 9, 7 if model != "RotatE" else 30
    ent, rel = _tables(model, E, R, k, rng, scale=0.3)
    t = _triples(E, R, B, rng)
    out = {}
    if model == "RotatE":  # its fast path has no dynamic assignment: this case covers the general kernel's
        monkeypatch.setenv("KGE_B200_TRAIN_KERNEL", "general")
    for mode in ("static", "dynamic"):
        monkeypatch.setenv("KGE_B200_TRAIN_SCHED", mode)
        # (a small step: RotatE's unit-vector gradients amplify atomic-order noise from one step to the next)
        eng = _engine(model, k, eta, E, R, loss="self_adversarial", optimizer="sgd", optimizer_params={"learning_rate": 1e-4})
        eng.set_embeddings(ent, rel)
        sp = torch.empty(B, device="cuda"); sn = torch.empty(eta * B, device="cuda")
        losses = []
        for step in range(3):
            eng.forward_backward(_dev(t), None, seed=5, step=step, scores_pos=sp, scores_neg=sn)
            if step == 0:
                first = (sp.cpu().numpy().copy(), sn.cpu().numpy().copy(), eng.g_ent.cpu().numpy().copy())
            eng.apply_gradients()
            losses.append(eng.read_loss())
        out[mode] = first + (_dense(eng, eng.ent), _dense(eng, eng.rel), losses)
        eng.close()
    a, b = out["static"], out["dynamic"]
    assert (a[0] == b[0]).all() and (a[1] == b[1]).all()
    assert _close(a[2], b[2], rtol=2e-5)
    assert np.allclose(a[5], b[5], rtol=1e-5), (a[5], b[5])  # every launch saw every positive exactly once
    assert _close(a[3], b[3], rtol=1e-4) and _close(a[4], b[4], rtol=1e-4)


@pytest.mark.parametrize("model,k,eta", [("RotatE", 200, 30), ("ComplEx", 600, 9), ("TransE", 300, 40)])
def test_single_buffered_groups_equal_prefetched_groups(model, k, eta, monkeypatch):
    """KGE_B200_TRAIN_NBUF=1 (a non-resident slot holds ONE group of corruptions, fetched on demand) against the default
    (two buffers, next group prefetched): same arithmetic per score, gradients to atomic-order noise."""
    rng = np.random.default_rng(89)
    E, R, B = 600, 5, 500
    ent, rel = _tables(model, E, R, k, rng, scale=0.3)
    t = _triples(E, R, B, rng)
    neg_ent, neg_keep = _negatives(E, B, eta, rng)
    out = {}
    for nbuf in ("2", "1"):
        monkeypatch.setenv("KGE_B200_TRAIN_NBUF", nbuf)
        eng = _engine(model, k, eta, E, R, loss="self_adversarial", neg_group=4)
        assert not eng.lib.kge_rows_resident(eng.h)
        eng.set_embeddings(ent, rel)
        sp = torch.empty(B, device="cuda"); sn = torch.empty(eta * B, device="cuda")
        eng.forward_backward(_dev(t), (_dev(neg_ent), _dev(neg_keep)), scores_pos=sp, scores_neg=sn)
        torch.cuda.synchronize()
        out[nbuf] = (sp.cpu().numpy(), sn.cpu().numpy(), eng.g_ent.cpu().numpy().copy(), eng.g_rel.cpu().numpy().copy(), eng.read_loss())
        eng.close()
    a, b = out["2"], out["1"]
    assert (a[0] == b[0]).all() and (a[1] == b[1]).all()
    assert _close(a[2], b[2], rtol=2e-5) and _close(a[3], b[3], rtol=2e-5)
    assert abs(a[4] - b[4]) <= 1e-6 * abs(a[4])


@pytest.mark.parametrize("model,k", [("TransE", 50), ("TransE", 403), ("RotatE", 7), ("RotatE", 200)])
def test_packed_pair_ranking_kernel_equals_scalar_tile_kernel(model, k, monkeypatch):
    """kge_rank_pair_kernel (two canonical chains per pair of fp32 registers) against kge_rank_tile_kernel (one chain per
    register, KGE_B200_RANK_KERNEL=tile): every corruption score bit for bit, ragged candidate / query counts, a window of
    candidates; both match the oracle elsewhere (test_corruption_scores_vs_oracle, the rank tests)."""
    rng = np.random.default_rng(97)
    E, R, b = 777, 6, 77
    ent, rel = _tables(model, E, R, k, rng, scale=0.7)
    ent[3] = ent[5]  # an exactly-zero residual on the object side of (3, p, 5)-style pairs: sqrt(0) must add exactly 0
    t = _triples(E, R, b, rng)
    t[0] = (3, 1, 5)
    eng = _engine(model, k, 1, E, R)
    eng.set_embeddings(ent, rel)
    for side in ("s", "o"):
        got = {}
        for kern in ("pair", "tile"):
            if kern == "tile":
                monkeypatch.setenv("KGE_B200_RANK_KERNEL", "tile")
            else:
                monkeypatch.delenv("KGE_B200_RANK_KERNEL", raising=False)
            full = eng.corruption_scores(_dev(t), side).cpu().numpy()
            win = eng.corruption_scores(_dev(t), side, cand_begin=100, n_cand=333).cpu().numpy()
            ranks = eng.rank(_dev(t), side, "middle").cpu().numpy()
            got[kern] = (full, win, ranks)
        for x, y in zip(got["pair"], got["tile"]):
            assert x.shape == y.shape and x.dtype == y.dtype, (model, k, side)
            bits = np.uint32 if x.dtype == np.float32 else x.dtype
            assert (x.view(bits) == y.view(bits)).all(), (model, k, side)
        assert (got["pair"][1] == got["pair"][0][:, 100:433]).all()
    eng.close()


def test_exchange_kernel_world1_equals_plain_optimizer():
    """kge_optimizer_step_exchange with world = 1 (peer pointers = own pointers, in-kernel flag barriers against itself)
    is the plain dense optimizer on the concatenated [ent|rel] block, zeroes the other gradient block and does not hang;
    the 2-GPU version of this check is tests/test_gpu_z_multi.py."""
    import ctypes as C
    from ampligraph_b200 import _lib
    rng = np.random.default_rng(61)
    model, E, R, k, eta, B = "ComplEx", 300, 7, 10, 3, 64
    ent, rel = _tables(model, E, R, k, rng, scale=0.5)
    regs = [{"p": 2, "lambda": 1e-3}, {"p": 3, "lambda": 1e-3}]
    kw = dict(loss="nll", optimizer="adam", optimizer_params={"learning_rate": 0.01}, regularizer=regs)
    ref = _engine(model, k, eta, E, R, **kw)
    ref.set_embeddings(ent, rel)
    eng = _engine(model, k, eta, E, R, **kw)
    ld, blk = eng.ld, E + R
    buf = torch.zeros((3 * blk + 1, ld), device="cuda")  # [ent|rel | g0 | g1 | flags]
    eng.ent, eng.rel = buf[0:E], buf[E:blk]
    eng.set_embeddings(ent, rel)
    gv = [(buf[blk:blk + E], buf[blk + E:2 * blk]), (buf[2 * blk:2 * blk + E], buf[2 * blk + E:3 * blk])]
    s0, s1 = torch.zeros((blk, ld), device="cuda"), torch.zeros((blk, ld), device="cuda")
    one = lambda ptr: (C.c_void_p * 1)(ptr)
    for step in range(4):
        t = _triples(E, R, B, rng)
        ne, nk = _negatives(E, B, eta, rng)
        b = step & 1
        eng.g_ent, eng.g_rel = gv[b]
        gv[b ^ 1][0].fill_(7.0)  # garbage in the OTHER block: the exchange must zero it
        eng.forward_backward(_dev(t), (_dev(ne), _dev(nk)))
        eng.t += 1
        _lib.check(eng.lib.kge_optimizer_step_exchange(
            eng.h, C.byref(eng.opt_cfgs["ent"]), C.byref(eng.opt_cfgs["rel"]), eng.t, 1, 0, one(buf.data_ptr()),
            one(gv[b][0].data_ptr()), None, None, C.c_void_p(gv[b ^ 1][0].data_ptr()), C.c_void_p(s0.data_ptr()), C.c_void_p(s1.data_ptr()),
            0, blk, one(buf[3 * blk:].data_ptr()), step + 1, 3, C.c_void_p(eng.loss_acc.data_ptr() + 8), eng._stream()))
        ref.train_step(_dev(t), (_dev(ne), _dev(nk)))
        torch.cuda.synchronize()
        assert (gv[b ^ 1][0] == 0).all() and (gv[b ^ 1][1] == 0).all()
    # same arithmetic element for element; the two engines' gradients differ only by the order of their fp32 atomics
    assert torch.allclose(eng.ent, ref.ent, rtol=1e-5, atol=1e-7) and torch.allclose(eng.rel, ref.rel, rtol=1e-5, atol=1e-7)
    got_loss, ref_loss = eng.read_loss(), ref.read_loss()  # read_loss() resets the accumulator: read each once
    assert abs(got_loss - ref_loss) <= 1e-6 * abs(ref_loss)
    eng.close(); ref.close()


# ---------------------------------------------------------------------------
def test_reference_rank_kats_on_gpu(kats):
    r = kats["ranks"]
    e_s, e_p, e_o = (np.array(r[x], np.float32) for x in ("e_s", "e_p", "e_o"))
    cand = np.array(r["ent_matrix"], np.float32)
    # entity table = candidates (ids 0..3) followed by the subject/object rows of the two test triples
    ent = np.concatenate([cand, e_s, e_o])
    n = len(e_s)
    t = np.stack([4 + np.arange(n), np.arange(n), 4 + n + np.arange(n)], 1).astype(np.int32)
    eng = _engine(r["model"], r["k"], 1, len(ent), n)
    eng.set_embeddings(ent, e_p)
    for case in r["cases"]:
        sides = [s for s in ("s", "o") if s in case["corrupt_side"]]
        got = []
        for j, side in enumerate(sides):
            off = idx = None
            if case["filters"]:
                f = case["filters"][j]
                off = _dev(np.concatenate([[0], np.cumsum([len(x) for x in f])]).astype(np.int64))
                idx = _dev(np.concatenate(f).astype(np.int32))
            got.append(eng.rank(_dev(t), side, case["comparison_type"], off, idx, cand_begin=0,
                                n_cand=case["end_ent_id"]).cpu().numpy())
        assert (np.array(got) == np.array(case["expected"], np.int32)).all(), (case, got)
    eng.close()


def _filters(E, b, rng, maxlen=8):
    lists = [sorted(set(rng.integers(0, E, rng.integers(0, maxlen)).tolist())) for _ in range(b)]
    off = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int64)
    idx = np.concatenate([np.asarray(x, np.int32) for x in lists]) if off[-1] else np.zeros(0, np.int32)
    return lists, off, idx.astype(np.int32)


@pytest.mark.parametrize("model", MODELS)
@pytest.mark.parametrize("k", [6, 50])
def test_ranks_bit_exact_vs_oracle(model, k):
    from oracle import c_oracle
    rng = np.random.default_rng(29)
    E, R, b = 700, 6, 70
    ent, rel = _tables(model, E, R, k, rng, scale=0.5)
    ent = np.round(ent, 2)  # coarse values -> plenty of quantisation ties
    t = _triples(E, R, b, rng)
    lists, off, idx = _filters(E, b, rng)
    eng = _engine(model, k, 1, E, R)
    eng.set_embeddings(ent, rel)
    for side in ("s", "o"):
        for strategy in ("worst", "best", "middle"):
            got = eng.rank(_dev(t), side, strategy).cpu().numpy()
            ref = c_oracle.rank_triples(model, side, strategy, ent, rel, t)
            assert (got == ref).all(), (model, side, strategy, np.flatnonzero(got != ref)[:5])
            gotf = eng.rank(_dev(t), side, strategy, _dev(off), _dev(idx)).cpu().numpy()
            reff = c_oracle.rank_triples(model, side, strategy, ent, rel, t, filters=lists)
            assert (gotf == reff).all(), (model, side, strategy, "filtered")
    eng.close()


@pytest.mark.parametrize("model", ["ComplEx", "RotatE", "TransE"])
def test_ranks_subset_and_shards(model):
    from oracle import c_oracle
    rng = np.random.default_rng(31)
    E, R, k, b = 1000, 5, 32, 40
    ent, rel = _tables(model, E, R, k, rng, scale=0.5)
    t = _triples(E, R, b, rng)
    eng = _engine(model, k, 1, E, R)
    eng.set_embeddings(ent, rel)
    # entities_subset (ScoringBasedEmbeddingModel.py:1634-1643): filter ids are subset positions
    subset = np.sort(rng.choice(E, 300, replace=False)).astype(np.int32)
    lists, off, idx = _filters(len(subset), b, rng)
    for side in ("s", "o"):
        got = eng.rank(_dev(t), side, "worst", _dev(off), _dev(idx), cand_ids=_dev(subset)).cpu().numpy()
        ref = c_oracle.rank_triples(model, side, "worst", ent, rel, t, filters=lists, cand_ids=subset)
        assert (got == ref).all()
    # row shards accumulate into the same output (ScoringBasedEmbeddingModel.py:1449-1452)
    lists, off, idx = _filters(E, b, rng)
    full = c_oracle.rank_triples(model, "o", "worst", ent, rel, t, filters=lists)
    out = torch.zeros(b, dtype=torch.int32, device="cuda")
    bounds = [0, 257, 600, E]
    for lo, hi in zip(bounds[:-1], bounds[1:]):
        eng.rank(_dev(t), "o", "worst", _dev(off), _dev(idx), cand_begin=lo, n_cand=hi - lo, out=out)
    assert (out.cpu().numpy() == full).all()
    eng.close()


def test_ranks_full_size_invariants():
    """cfg2 table size, 1,024 queries: worst >= middle >= best, filtered <= unfiltered,
    shard additivity, and a 64-query slice bit-exact against the oracle."""
    from oracle import c_oracle
    rng = np.random.default_rng(37)
    model, E, R, k, b = "ComplEx", 14505, 237, 200, 1024
    eng = _engine(model, k, 1, E, R)
    eng.init_glorot_uniform(seed=3)
    t = _triples(E, R, b, rng)
    lists, off, idx = _filters(E, b, rng, maxlen=40)
    td = _dev(t)
    w = eng.rank(td, "s", "worst").cpu().numpy()
    m = eng.rank(td, "s", "middle").cpu().numpy()
    be = eng.rank(td, "s", "best").cpu().numpy()
    wf = eng.rank(td, "s", "worst", _dev(off), _dev(idx)).cpu().numpy()
    assert (w >= m).all() and (m >= be).all() and (wf <= w).all() and (w >= 1).all()
    out = torch.zeros(b, dtype=torch.int32, device="cuda")
    for lo, hi in ((0, 5000), (5000, 9999), (9999, E)):
        eng.rank(td, "s", "worst", _dev(off), _dev(idx), cand_begin=lo, n_cand=hi - lo, out=out)
    assert (out.cpu().numpy() == wf).all()
    ent, rel = (x.cpu().numpy() for x in eng.get_embeddings())
    ref = c_oracle.rank_triples(model, "s", "worst", ent, rel, t[:64], filters=lists[:64])
    assert (wf[:64] == ref).all()
    eng.close()


def test_scoring_layer_plugin_methods_on_reference_kats(kats):
    """SCORING_LAYER_REGISTRY[name](k) exposes the reference's plugin methods (AbstractScoringLayer.py:103-156) on
    EMBEDDINGS: _compute_scores and the diagonal of both corruption-score matrices reproduce the reference's golden
    vectors (test_TransE.py:15-46 etc.), get_ranks its rank KATs (test_AbstractScoringLayer.py:15-53)."""
    from ampligraph_b200.latent_features import SCORING_LAYER_REGISTRY
    for c in kats["scoring"]:
        layer = SCORING_LAYER_REGISTRY[c["model"]](c["k"])
        if c["model"] == "RotatE":
            layer.max_rel_size = c["max_rel_size"]
        e_s, e_p, e_o = (np.array(c[x], np.float32) for x in ("e_s", "e_p", "e_o"))
        want = np.array(c["expected"], np.float32)
        if c["form"] == "triple":
            got = layer._compute_scores([e_s, e_p, e_o])
        elif c["form"] == "sub_diag":
            got = np.diag(layer._get_subject_corruption_scores([e_s, e_p, e_o], np.array(c["ent_matrix"], np.float32)))
        else:
            got = np.diag(layer._get_object_corruption_scores([e_s, e_p, e_o], np.array(c["ent_matrix"], np.float32)))
        assert (np.around(got, c["round_decimals"]) == want).all(), (c["source"], got, want)
    r = kats["ranks"]
    layer = SCORING_LAYER_REGISTRY[r["model"]](r["k"])
    e_s, e_p, e_o = (np.array(r[x], np.float32) for x in ("e_s", "e_p", "e_o"))
    cand = np.array(r["ent_matrix"], np.float32)
    for case in r["cases"]:
        got = layer.get_ranks([e_s, e_p, e_o], cand, case["start_ent_id"], case["end_ent_id"], case["filters"] or [],
                              None, case["corrupt_side"], case["comparison_type"])
        assert (got == np.array(case["expected"], np.int32)).all(), (case, got)


@pytest.mark.parametrize("model", MODELS)
def test_corruption_scores_vs_oracle(model):
    """kge_corruption_scores: the [b, n_cand] matrix, bit-identical to the oracle's canonical chain, subset and range forms."""
    from oracle import c_oracle
    rng = np.random.default_rng(67)
    E, R, k, b = 333, 5, 21, 37
    ent, rel = _tables(model, E, R, k, rng, scale=0.5)
    t = _triples(E, R, b, rng)
    eng = _engine(model, k, 1, E, R)
    eng.set_embeddings(ent, rel)
    sub = np.sort(rng.choice(E, 50, replace=False)).astype(np.int32)
    for side in ("s", "o"):
        ref = c_oracle.corruption_scores(model, side, ent[t[:, 0]], rel[t[:, 1]], ent[t[:, 2]], ent, max_rel_size=R)
        got = eng.corruption_scores(_dev(t), side).cpu().numpy()
        assert got.shape == (b, E) and (got == ref).all(), np.abs(got - ref).max()
        got = eng.corruption_scores(_dev(t), side, cand_begin=100, n_cand=77).cpu().numpy()
        assert (got == ref[:, 100:177]).all()
        got = eng.corruption_scores(_dev(t), side, cand_ids=_dev(sub)).cpu().numpy()
        assert (got == ref[:, sub]).all()
    eng.close()


def test_middle_strategy_over_candidate_partitions():
    """ADVICE r1: 'middle' = greater + ceil(equal/2) is not additive over candidate partitions; accumulating the RAW
    counters and finalizing once is (this is what the row-sharded paths do).  Coarse scores -> many ties."""
    from oracle import c_oracle
    rng = np.random.default_rng(71)
    model, E, R, k, b = "DistMult", 500, 3, 4, 64
    ent = np.round(rng.uniform(-1, 1, (E, k)), 1).astype(np.float32)
    rel = np.round(rng.uniform(-1, 1, (R, k)), 1).astype(np.float32)
    t = _triples(E, R, b, rng)
    lists, off, idx = _filters(E, b, rng)
    eng = _engine(model, k, 1, E, R)
    eng.set_embeddings(ent, rel)
    for strategy in ("middle", "worst", "best"):
        want = c_oracle.rank_triples(model, "o", strategy, ent, rel, t, filters=lists)
        counts = torch.zeros((b, 3), dtype=torch.int32, device="cuda")
        for lo, hi in ((0, 101), (101, 333), (333, E)):
            eng.rank(_dev(t), "o", strategy, _dev(off), _dev(idx), cand_begin=lo, n_cand=hi - lo, counts=counts)
        got = eng.finalize_ranks(counts, strategy).cpu().numpy()
        assert (got == want).all(), strategy
    # the naive accumulation really is wrong for 'middle' on this input (so the test above has teeth)
    naive = torch.zeros(b, dtype=torch.int32, device="cuda")
    for lo, hi in ((0, 101), (101, 333), (333, E)):
        eng.rank(_dev(t), "o", "middle", _dev(off), _dev(idx), cand_begin=lo, n_cand=hi - lo, out=naive)
    assert (naive.cpu().numpy() != c_oracle.rank_triples(model, "o", "middle", ent, rel, t, filters=lists)).any()
    eng.close()


def test_two_handles_two_streams_device_guard():
    """Every entry point makes its handle's device current and restores the caller's (ADVICE r1 low): drive a handle
    from a thread whose current device is changed underneath, on a non-default stream."""
    rng = np.random.default_rng(73)
    E, R, k = 50, 3, 6
    ent, rel = _tables("TransE", E, R, k, rng, scale=0.5)
    eng = _engine("TransE", k, 1, E, R)
    eng.set_embeddings(ent, rel)
    t = _dev(_triples(E, R, 20, rng))
    want = eng.score(t).cpu()
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        got = eng.score(t)
    st.synchronize()
    assert torch.equal(got.cpu(), want) and torch.cuda.current_device() == 0
    eng.close()


TC_MODELS = ["DistMult", "ComplEx", "HolE"]


@pytest.mark.parametrize("model,k,E,b,scale", [("ComplEx", 200, 3000, 200, 0.05), ("DistMult", 400, 2100, 130, 0.3),
                                               ("HolE", 37, 1500, 70, 0.5), ("ComplEx", 1000, 800, 257, 0.02),
                                               ("DistMult", 50, 5000, 64, 1.0)])
def test_tc_filter_error_bound(model, k, E, b, scale):
    """The tensor-core filter pass (wgmma, split-bf16 operands) is sound iff its approximate score is within the bound it
    assumes of the canonical FP32 score for EVERY (query, candidate) pair (kge_rank_tc.cu header).  Measured through
    kge_rank_filter_probe against kge_corruption_scores; the bound must also hold with a >= 4x margin, and the
    approximation must be genuinely fine (3 bf16 products, not 1)."""
    rng = np.random.default_rng(83)
    R = 9
    ent, rel = _tables(model, E, R, k, rng, scale=scale)
    t = _triples(E, R, b, rng)
    eng = _engine(model, k, 1, E, R, rank_mode="auto")
    eng.set_embeddings(ent, rel)
    for side in ("s", "o"):
        exact = eng.corruption_scores(_dev(t), side)
        approx, delta = eng.rank_filter_probe(_dev(t), side)
        err = (approx.double() - exact.double()).abs()
        assert bool((delta > 0).all()) and bool((err <= delta.double()).all()), float((err / delta.double()).max())
        worst = float((err / delta.double()).max())
        assert worst <= 0.25, worst
        rel_err = float(err.max() / exact.abs().max())
        assert rel_err < 2e-5, rel_err   # a single bf16 product would sit at ~4e-3
    eng.close()


@pytest.mark.parametrize("model", TC_MODELS)
@pytest.mark.parametrize("E,b,k,coarse", [(5000, 300, 50, True), (1300, 129, 200, False), (20000, 1024, 24, True)])
def test_ranks_tensor_core_filter_equals_exact_chain(model, E, b, k, coarse):
    """KGE_RANK_MODE_AUTO (tensor-core filter + exact refine) == KGE_RANK_MODE_EXACT (canonical FP32 chain for every
    pair), bit for bit: both sides, all three tie strategies, filtered and unfiltered, candidate ranges and subsets,
    raw counters.  Coarse tables put thousands of candidates exactly ON the positive's bin (ties), fine ones next to it."""
    rng = np.random.default_rng(89)
    R = 7
    ent, rel = _tables(model, E, R, k, rng, scale=0.6)
    if coarse:
        ent, rel = np.round(ent, 1), np.round(rel, 1)
    t = _triples(E, R, b, rng)
    lists, off, idx = _filters(E, b, rng, maxlen=12)
    a = _engine(model, k, 1, E, R, rank_mode="auto")
    x = _engine(model, k, 1, E, R, rank_mode="exact")
    a.set_embeddings(ent, rel); x.set_embeddings(ent, rel)
    td = _dev(t)
    sub = _dev(np.sort(rng.choice(E, 777, replace=False)).astype(np.int32))
    for side in ("s", "o"):
        for strategy in ("worst", "best", "middle"):
            assert torch.equal(a.rank(td, side, strategy), x.rank(td, side, strategy)), (side, strategy)
        assert torch.equal(a.rank(td, side, "worst", _dev(off), _dev(idx)), x.rank(td, side, "worst", _dev(off), _dev(idx)))
        assert torch.equal(a.rank(td, side, "worst", cand_begin=123, n_cand=E - 200), x.rank(td, side, "worst", cand_begin=123, n_cand=E - 200))
        assert torch.equal(a.rank(td, side, "middle", cand_ids=sub), x.rank(td, side, "middle", cand_ids=sub))
        ca = torch.zeros((b, 3), dtype=torch.int32, device="cuda"); cx = torch.zeros_like(ca)
        a.rank(td, side, "worst", _dev(off), _dev(idx), counts=ca); x.rank(td, side, "worst", _dev(off), _dev(idx), counts=cx)
        assert torch.equal(ca, cx)
    a.close(); x.close()


def test_tensor_core_filter_overflow_falls_back_to_exact():
    """When more pairs are undecided than the list holds, the gated exact kernel recounts the whole call: same ranks."""
    from oracle import c_oracle
    rng = np.random.default_rng(97)
    model, E, R, k, b = "DistMult", 1500, 3, 8, 96
    ent = np.round(rng.uniform(-1, 1, (E, k)), 1).astype(np.float32)
    rel = np.round(rng.uniform(-1, 1, (R, k)), 1).astype(np.float32)
    t = _triples(E, R, b, rng)
    eng = _engine(model, k, 1, E, R, rank_mode="auto", rank_pair_cap=5)  # thousands of exact ties -> far more than 5 undecided pairs
    eng.set_embeddings(ent, rel)
    for side in ("s", "o"):
        got = eng.rank(_dev(t), side, "middle").cpu().numpy()
        assert (got == c_oracle.rank_triples(model, side, "middle", ent, rel, t)).all()
    eng.close()


def test_error_convention():
    from ampligraph_b200 import _lib
    with pytest.raises(ValueError):
        _engine("NoSuchModel", 4, 1, 10, 2)
    with pytest.raises(ValueError):
        _engine("TransE", 4, 1, 10, 2, loss="nope")
    eng = _engine("TransE", 4, 1, 10, 2)
    with pytest.raises(ValueError):  # invalid corrupt side id
        _lib.check(eng.lib.kge_rank(eng.h, 7, 0, None, None, None, 0, None, 0, 0, None, None, 0, None, None, None, 0, None))
    with pytest.raises(ValueError):  # the workspace is the caller's: too small -> refused, never allocated behind its back
        out = torch.zeros(4, dtype=torch.int32, device="cuda")
        tr = torch.zeros((4, 3), dtype=torch.int32, device="cuda")
        ws = torch.empty(4096, dtype=torch.uint8, device="cuda")
        ws = ws[(-ws.data_ptr()) % 1024:]
        _lib.check(eng.lib.kge_rank(eng.h, 0, 0, eng.ent.data_ptr(), eng.rel.data_ptr(), tr.data_ptr(), 4, None, 0, 10, None,
                                    None, 0, out.data_ptr(), None, ws.data_ptr(), 8, None))
    assert eng.lib.kge_rank_workspace_bytes(eng.h, 4, 10) > 8
    with pytest.raises(ValueError):  # gradient buffers are mandatory outside FORWARD_ONLY
        _lib.check(eng.lib.kge_train_step(eng.h, 0, eng.ent.data_ptr(), eng.rel.data_ptr(), None, None,
                                          eng.ent.data_ptr(), 1, None, None, 0, 0, None, None, None, None, None, None))
    eng.close()
