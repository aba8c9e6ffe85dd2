"""Oracle of embedding dropout in the all-candidate steps (kge_set_embedding_dropout, DESIGN.md 3.19).  Test
infrastructure only.

- The mask stream, in plain Python on oracle/philox.py (mask_words), and the same in numpy (philox_np), which the host
  tests check against it: element c of row `row` under tag = 4 side + role takes word c & 3 of
  philox4x32_10((row, (c >> 2) | (0x80 | tag) << 24, step_lo, step_hi), (seed_lo, seed_hi)) and is kept iff
  (word >> 8) >= round(p 2^24).  c is the column of the kernel's padded row (each half padded to 4 floats).
- The float64 step of one side on the dropped copies: the candidates' dropped table and each query occurrence's dropped
  rows are the leaves, the loss is the side's oracle loss (one_vs_all_oracle / k_vs_all_oracle / relation_prediction_
  oracle), and each leaf's gradient maps back to its raw row through scale * m.
- The per-element bound of exact_oracle.OvaBound for the same step, formed on the |raw tables| through the masks, so
  that it lands on the raw elements, plus one rounding for the final fp32(scale * g~)."""
import numpy as np
import torch

import exact_oracle as xo
import k_vs_all_oracle
import one_vs_all_oracle
import relation_prediction_oracle
from oracle import philox, ref_step

MASK = 0xFFFFFFFF
SIDE = {"s": 1, "o": 2, "p": 3}


def tag(side, role):
    """role 0: the candidate rows; 1 + j: the query's triple column j."""
    return 4 * SIDE[side] + role


def threshold(p):
    """round(p 2^24) of the fp32 p, halves away from zero (llround)."""
    return int(np.floor(float(np.float32(p)) * 2.0 ** 24 + 0.5))


def scale(p):
    return np.float32(1.0 / (1.0 - float(np.float32(p))))


def mask_words(seed, step, tg, row, c):
    """The 32-bit word of element c of row `row` under tag tg (plain Python on oracle/philox.py)."""
    ctr = (row & MASK, (c >> 2) | ((0x80 | tg) << 24), step & MASK, step >> 32)
    return philox.philox4x32_10(ctr, (seed & MASK, seed >> 32))[c & 3]


def philox_np(c0, c1, c2, c3, k0, k1):
    """philox4x32_10 on uint64 arrays holding 32-bit lanes (broadcast) -> the four output lanes."""
    M0, M1, W0, W1 = np.uint64(philox.M0), np.uint64(philox.M1), np.uint64(philox.W0), np.uint64(philox.W1)
    m, s32 = np.uint64(MASK), np.uint64(32)
    c0, c1, c2, c3, k0, k1 = [np.asarray(x, np.uint64) & m for x in (c0, c1, c2, c3, k0, k1)]
    for _ in range(10):
        p0, p1 = M0 * c0, M1 * c2
        c0, c1, c2, c3 = (p1 >> s32) ^ c1 ^ k0, p1 & m, (p0 >> s32) ^ c3 ^ k1, p0 & m
        k0, k1 = (k0 + W0) & m, (k1 + W1) & m
    return c0, c1, c2, c3


def words(seed, step, tg, rows, ld):
    """[len(rows), ld] uint64 mask words of the given row keys, columns 0 .. ld - 1 of the padded row."""
    rows = np.asarray(rows, np.uint64).reshape(-1, 1)
    blk = np.arange(ld // 4, dtype=np.uint64).reshape(1, -1)
    out = philox_np(rows, blk | np.uint64((0x80 | tg) << 24), step & MASK, step >> 32, seed & MASK, seed >> 32)
    return np.stack(out, 2).reshape(rows.shape[0], ld)


def keep(seed, step, tg, rows, ld, p):
    return (words(seed, step, tg, rows, ld) >> np.uint64(8)) >= np.uint64(threshold(p))


def padded_columns(model, K):
    """The padded-row column of each of the K dense columns (each half padded to a multiple of 4 floats)."""
    if model == "DistMult":
        return np.arange(K)
    h, kp = K // 2, -(-(K // 2) // 4) * 4
    return np.concatenate([np.arange(h), kp + np.arange(h)])


def dense_keep(model, K, seed, step, tg, rows, p):
    """The mask of dense [len(rows), K] rows."""
    ld = xo.row_stride(model, K)
    return keep(seed, step, tg, rows, ld, p)[:, padded_columns(model, K)]


class Dropout:
    """(p_ent, p_rel, seed, step) of a step."""

    def __init__(self, p_ent, p_rel, seed, step):
        self.p = {"e": p_ent, "r": p_rel}
        self.seed, self.step = int(seed), int(step)

    def factor(self, model, K, side, role, rows, table):
        """[len(rows), K] float64 scale * m of rows `rows` of `table` ('e' / 'r') under (side, role)."""
        p = self.p[table]
        m = dense_keep(model, K, self.seed, self.step, tag(side, role), rows, p)
        return m * float(scale(p))

    def dropped(self, x, f):
        """fp32(x * scale) where kept, +0 where dropped (f = factor)."""
        x = np.asarray(x, np.float32)
        s = np.float32(f.max()) if f.max() > 0 else np.float32(1.0)
        return np.where(f > 0, x * s, np.float32(0.0)).astype(np.float32)


def _side_parts(model, side, ent, rel, t, dr):
    """For one side: (cand_table_key, cand_factor [n_cand, K], query parts [(table key, triple column, raw rows, factor)])."""
    K = ent.shape[1]
    B = t.shape[0]
    b = np.arange(B)
    if side == "p":
        cand_key, cand_raw = "r", rel
        cols = (0, 2)
    else:
        cand_key, cand_raw = "e", ent
        cols = (0, 1) if side == "o" else (1, 2)
    fc = dr.factor(model, K, side, 0, np.arange(cand_raw.shape[0]), cand_key)
    parts = []
    for j in cols:
        key = "r" if j == 1 else "e"
        raw = (rel if key == "r" else ent)[t[:, j]]
        parts.append((key, j, raw, dr.factor(model, K, side, 1 + j, b, key)))
    return cand_key, cand_raw, fc, parts


def _query(model, side, a, c):
    """The side's query from its two query rows (a, c) in triple-column order."""
    if side == "p":
        return relation_prediction_oracle.relation_query(model, a, c)
    if side == "o":
        return one_vs_all_oracle.query_vectors(model, "o", a, c, c)
    return one_vs_all_oracle.query_vectors(model, "s", a, a, c)  # side s reads (p, o) only


def _side_loss(logits, side, t, reduction, weight, labels, eps):
    if labels is not None:
        y = k_vs_all_oracle.targets(labels, logits.shape[1], eps)
        return k_vs_all_oracle.side_loss(logits, y, reduction).sum()
    target = torch.as_tensor(t[:, {"s": 0, "o": 2, "p": 1}[side]], dtype=torch.long)
    return weight * one_vs_all_oracle.side_loss(logits, target, reduction).sum()


def side_step(model, ent, rel, triples, side, dr, reduction="sum", weight=1.0, labels=None, eps=0.0):
    """(loss, g_ent, g_rel, logits) of one side under dropout dr, float64; labels: KvsAll."""
    ent, rel = np.asarray(ent, np.float32), np.asarray(rel, np.float32)
    t = np.asarray(triples, np.int64).reshape(-1, 3)
    cand_key, cand_raw, fc, parts = _side_parts(model, side, ent, rel, t, dr)
    C = torch.tensor(dr.dropped(cand_raw, fc), dtype=torch.float64, requires_grad=True)
    Q = [torch.tensor(dr.dropped(raw, f), dtype=torch.float64, requires_grad=True) for _, _, raw, f in parts]
    logits = _query(model, side, Q[0], Q[1]) @ C.T
    loss = _side_loss(logits, side, t, reduction, weight, labels, eps)
    loss.backward()
    g = {"e": np.zeros(ent.shape, np.float64), "r": np.zeros(rel.shape, np.float64)}
    g[cand_key] += fc * C.grad.numpy()
    for (key, j, _, f), q in zip(parts, Q):
        np.add.at(g[key], t[:, j], f * q.grad.numpy())
    return float(loss.detach()), g["e"], g["r"], logits.detach()


class DropoutBound(xo.OvaBound):
    """exact_oracle.OvaBound of steps under dropout: the same weights per (query, candidate) pair, with the |query| and
    |candidate| rows formed through the masks from the |raw tables| (so the bound lands on the raw elements), and one
    more rounding per element for the final fp32(scale * g~) (check)."""

    def add_dropout_side(self, queries, side, dr, reduction="sum", weight=1.0, labels=None, eps=0.0):
        u, model = xo.FP32_EPS, self.model
        t = np.asarray(queries, np.int64).reshape(-1, 3)
        B = t.shape[0]
        ent, rel = self.E.numpy().astype(np.float32), self.R.numpy().astype(np.float32)
        cand_key, cand_raw, fc, parts = _side_parts(model, side, ent, rel, t, dr)
        tab = {"e": (self.E, self.Ea), "r": (self.R, self.Ra)}
        X = torch.tensor(dr.dropped(cand_raw, fc), dtype=torch.float64)
        Xa = tab[cand_key][1] * torch.as_tensor(fc)
        qrows = [torch.tensor(dr.dropped(raw, f), dtype=torch.float64) for _, _, raw, f in parts]
        arows = [tab[key][1][torch.as_tensor(t[:, j])] * torch.as_tensor(f) for key, j, _, f in parts]
        q = _query(model, side, qrows[0], qrows[1])
        qa = xo.abs_query(model, arows[0], arows[1])  # side o: (s, p); side s: (p, o); side p: (s, o)
        n_cand = X.shape[0]
        ns, xs = xo.ova_geometry(B, n_cand, side == "p")
        n, n_loss = xo.ova_chains(B, n_cand, ns, xs, labels is not None)
        n = n + self.n_red + xo.OVA_C
        logits = (q @ X.T).detach()
        AS = qa @ Xa.T
        lam = (self.ld + 4) * u * AS.detach()
        inr = (logits.abs() <= ref_step.CLIP_HI).double()
        near = ((logits.abs() - ref_step.CLIP_HI).abs() < lam).double()
        lg = logits.clone().requires_grad_(True)
        g = torch.autograd.grad(_side_loss(lg, side, t, reduction, weight, labels, eps), lg)[0].abs()
        if labels is None:
            target = torch.as_tensor(t[:, {"s": 0, "o": 2, "p": 1}[side]])
            lc, P, m, D = one_vs_all_oracle.side_softmax(logits, target, reduction)
            P = weight * P
            T = torch.zeros_like(P).scatter_(1, target[:, None], weight)
            G = (P * (m - lc)).sum(1, keepdim=True) / weight
            W = (inr * ((g + P) * n + P * ((lam + lam.max(1, keepdim=True).values) / u + (lc - m).abs() + 3 * G))
                 + near * (g + P + T) / u)
            lt = lc.gather(1, target[:, None])
            self.loss += weight * float(((n_loss + xo.OVA_C) * u * (1 + m.abs() + torch.log(D).abs() + lt.abs())
                                         + lam.max(1, keepdim=True).values + lam.gather(1, target[:, None])).sum())
        else:
            w = 1.0 / n_cand if reduction == "mean" else 1.0
            y = k_vs_all_oracle.targets(labels, n_cand, eps)
            lc = torch.clamp(logits, ref_step.CLIP_LO, ref_step.CLIP_HI)
            sig = torch.sigmoid(lc)
            W = inr * (g * n + w * (sig * (1 - sig) * lam / u + xo.OVA_C)) + near * (g + w * (sig - y).abs()) / u
            sp = torch.nn.functional.softplus(lc)
            self.loss += w * float(((n_loss + xo.OVA_C) * u * (sp + (y * lc).abs()) + lam * (sig - y).abs()).sum())
        for acc, wt in ((self.A, W), (self.A1, torch.ones_like(W))):
            self.Ea.grad = self.Ra.grad = None
            (wt * AS).sum().backward(retain_graph=True)
            acc[0] += self.Ea.grad
            acc[1] += self.Ra.grad

    def check(self, got_ent, got_rel, want_ent, want_rel, where=""):
        for name, got, want, A, A1 in (("g_ent", got_ent, want_ent, self.A[0], self.A1[0]),
                                       ("g_rel", got_rel, want_rel, self.A[1], self.A1[1])):
            got = torch.as_tensor(np.asarray(got), dtype=torch.float64)
            want = torch.as_tensor(np.asarray(want), dtype=torch.float64)
            assert bool(torch.isfinite(got).all()), (where, name)
            ok, ratio = xo.within_bound(got, want, A, A1, 1 - 8, 1)  # + the final fp32(scale * g~)
            assert ok, (where, name, "worst error / bound %.3g" % ratio)
