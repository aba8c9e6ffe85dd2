"""The per-element bound of the predict path (exact_oracle.PredictBound) on the host: it is sound for a restatement of
kge_score_kernel's exact fp32 operation order, not vacuous, and sharp enough to reject that restatement with one defect.

The restatement follows kge_misc.cu: one warp per triple, lane l's register chain over columns l, l + 32, ... < k
(fmaf correctly rounded through optim_exact_oracle.fma32, every other operation numpy float32, which rounds as the
library's non-fast-math build does, subnormals kept), the xor butterfly of warp_sum, and lane 0's scale * acc with
scale = fl(2 / k) for HolE."""
import numpy as np
import pytest
import torch

import exact_oracle as xo
from optim_exact_oracle import fma32

F = np.float32
MODELS = ["TransE", "DistMult", "ComplEx", "HolE", "RotatE"]
KS = [1, 5, 33, 100]
FLOOR = 0.02  # the worst error / bound each restated model reaches at k = 100 over the three table kinds


def kernel_scores(model, ent, rel, triples, max_rel_size=None, defect=None):
    """kge_score_kernel in numpy fp32 on dense tables (RotatE: rel is the theta table; the kernel reads its fp32
    rotation table).  defect: None, 'tail' (the columns past the last full 32-column window dropped), 'lane' (lane 3's
    chain added twice) or 'scale' (HolE's fl(2 / k) applied twice)."""
    t = np.asarray(triples)
    K = ent.shape[1]
    k = K if model in ("TransE", "DistMult") else K // 2
    S, O = ent[t[:, 0]].astype(F), ent[t[:, 2]].astype(F)
    if model == "RotatE":
        c, sn = xo.rotation_table(rel[:, :k], xo.rotation_divisor32(K, max_rel_size or rel.shape[0])[0])
        P = np.concatenate([c, sn], 1)[t[:, 1]].astype(F)
    else:
        P = rel[t[:, 1]].astype(F)
    acc = np.zeros((len(t), 32), F)
    stop = k - k % 32 if defect == "tail" else k
    with np.errstate(all="ignore"):
        for base in range(0, stop, 32):
            d = np.arange(base, min(base + 32, stop))
            a = acc[:, :len(d)]
            if model == "TransE":
                a = a - np.abs((S[:, d] + P[:, d]) - O[:, d])
            elif model == "DistMult":
                a = fma32(S[:, d] * P[:, d], O[:, d], a)
            elif model in ("ComplEx", "HolE"):
                sr, si, pr, pi, orr, oi = S[:, d], S[:, k + d], P[:, d], P[:, k + d], O[:, d], O[:, k + d]
                a = fma32(sr, fma32(pi, oi, pr * orr), a)
                a = fma32(si, fma32(-pi, orr, pr * oi), a)
            else:
                sr, si, c, sn = S[:, d], S[:, k + d], P[:, d], P[:, k + d]
                re = fma32(-si, sn, sr * c) - O[:, d]
                im = fma32(si, c, sr * sn) - O[:, k + d]
                a = a - np.sqrt(fma32(im, im, re * re))
            acc[:, :len(d)] = a
        if defect == "lane":
            acc[:, 3] = acc[:, 3] + acc[:, 3]
        lanes = np.arange(32)
        for off in (16, 8, 4, 2, 1):
            acc = acc + acc[:, lanes ^ off]
        scale = F(2.0 / k) if model == "HolE" else F(1.0)
        out = scale * acc[:, 0]
        if defect == "scale":
            out = scale * out
    assert out.dtype == F
    return out


def glorot(rng, rows, K):
    lim = np.sqrt(6.0 / (rows + K))
    return rng.uniform(-lim, lim, (rows, K)).astype(F)


def tables(model, k, kind, rng, E=400, R=9, n=600):
    """(ent, rel, triples).  'glorot'; 'scaled': every row times 2^e, e uniform in [-20, 20] (RotatE: entity rows
    only, the phases stay in range); 'cancel': the object row makes the score nearly cancel -- the trilinear models'
    o is a random row minus its projection on the query d score / d o, TransE's o = s + p and RotatE's o = R(phi) s,
    each plus noise 2^-12 of its size, so |score| is far below |score|_abs; 'subnormal': a tenth of the rows hold
    subnormal entries in half their columns."""
    K = xo.internal_k(model, k)
    ent, rel = glorot(rng, E, K), glorot(rng, R, K)
    t = np.stack([rng.integers(0, E, n), rng.integers(0, R, n), rng.integers(0, E, n)], 1).astype(np.int32)
    if kind == "scaled":
        ent *= (2.0 ** rng.integers(-20, 21, E))[:, None].astype(F)
        if model != "RotatE":
            rel *= (2.0 ** rng.integers(-20, 21, R))[:, None].astype(F)
    elif kind == "subnormal":
        for tab, rows in ((ent, E), (rel, R if model != "RotatE" else 0)):
            for r in (rng.choice(rows, max(1, rows // 10), replace=False) if rows else []):
                cols = rng.random(K) < 0.5
                tab[r, cols] = (rng.uniform(-1, 1, int(cols.sum())) * 2.0 ** -126).astype(F)
    elif kind == "cancel":  # rows [0, n) are the objects, one per triple; the subjects come from [n, E)
        assert 2 * n <= E
        t[:, 0], t[:, 2] = rng.integers(n, E, n), np.arange(n)
        Et, Rt = torch.as_tensor(ent, dtype=torch.float64), torch.as_tensor(rel, dtype=torch.float64)
        s, p = Et[t[:, 0]], Rt[t[:, 1]]
        if model in xo.TRILINEAR:
            w = Et[t[:, 2]].clone().requires_grad_(True)
            xo.scores(model, s, p, w).sum().backward()
            q = w.grad
            o = w.detach() - ((w.detach() * q).sum(1, keepdim=True) / (q * q).sum(1, keepdim=True)) * q
        elif model == "TransE":
            o = s + p
        else:
            h = K // 2
            c, sn = xo.rotation_table(rel[:, :h], xo.rotation_divisor32(K, R)[0])
            c, sn = torch.as_tensor(c, dtype=torch.float64)[t[:, 1]], torch.as_tensor(sn, dtype=torch.float64)[t[:, 1]]
            o = torch.cat([s[:, :h] * c - s[:, h:] * sn, s[:, :h] * sn + s[:, h:] * c], 1)
        o = o * (1 + 2.0 ** -12 * torch.as_tensor(rng.uniform(-1, 1, o.shape)))
        ent[t[:, 2]] = o.numpy().astype(F)
    return ent, rel, t


def run(model, k, kind, seed=0, defect=None):
    rng = np.random.default_rng(seed)
    ent, rel, t = tables(model, k, kind, rng, E=800 if kind == "cancel" else 400, n=400 if kind == "cancel" else 600)
    bound = xo.PredictBound(model, ent, rel, t)
    return bound, kernel_scores(model, ent, rel, t, defect=defect)


@pytest.mark.parametrize("kind", ["glorot", "scaled", "cancel", "subnormal"])
@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("model", MODELS)
def test_restated_kernel_within_bound(model, k, kind):
    """Every score of the restated kernel lies within the bound, and is finite."""
    bound, got = run(model, k, kind)
    assert np.isfinite(got).all()
    ok, ratio, i = bound.check(got)
    print("\n%s k=%d %s: worst error / bound %.4f" % (model, k, kind, ratio))
    assert ok, (model, k, kind, ratio, i)


@pytest.mark.parametrize("model", MODELS)
def test_bound_is_not_vacuous(model):
    """The worst error / bound over the three real-valued table kinds at k = 100 reaches FLOOR: the bound is within a
    small factor of what the kernel's order of operations actually loses."""
    worst = max(bound.check(got)[1] for bound, got in (run(model, 100, kind, seed)
                                                         for kind in ("glorot", "scaled", "cancel") for seed in (0, 1)))
    print("\n%s: worst error / bound %.4f" % (model, worst))
    assert worst >= FLOOR, worst


DEFECTS = [(m, k, "tail") for m in MODELS for k in (5, 33, 100)] + [(m, k, "lane") for m in MODELS for k in (5, 100)] + \
          [("HolE", k, "scale") for k in (1, 5, 100)]


@pytest.mark.parametrize("model,k,defect", DEFECTS)
def test_bound_rejects_one_defect(model, k, defect):
    """The restatement with one defect fails the bound: the columns of the last, partial window dropped (k % 32 != 0),
    one lane's chain counted twice, HolE's scale applied twice."""
    bound, got = run(model, k, "glorot", defect=defect)
    ok, ratio, _ = bound.check(got)
    assert not ok, (model, k, defect, ratio)


def test_nonfinite_classes():
    """+-inf and NaN entries: the restated kernel's NaN / +inf / -inf pattern is the float64 oracle's, and check
    compares it exactly (a finite score where the oracle's is infinite fails)."""
    rng = np.random.default_rng(3)
    for model in MODELS:
        ent, rel, t = tables(model, 33, "glorot", rng)
        for v, r in zip((np.inf, -np.inf, np.nan, np.inf), rng.choice(len(ent), 4, replace=False)):
            ent[r, rng.integers(0, ent.shape[1])] = v
        if model != "RotatE":
            rel[1, 0] = np.inf
        bound = xo.PredictBound(model, ent, rel, t)
        got = kernel_scores(model, ent, rel, t)
        ok, ratio, i = bound.check(got)
        assert ok and not np.isfinite(got).all(), (model, ratio, i)
        bad = got.copy()
        j = int(np.nonzero(~np.isfinite(got))[0][0])
        bad[j] = 0.0
        assert not bound.check(bad)[0], model
