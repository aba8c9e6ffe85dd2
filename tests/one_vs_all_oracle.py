"""Float64 oracle of 1vsAll training (kge_one_vs_all_step, DESIGN.md 3.12): the multiclass NLL of every positive
against every entity, with the gradients of both tables from torch autograd.  The all-entity scores are
oracle.ref_step.corruption_scores (the reference's broadcast form) for small cases, or the same scores as one matrix
product (matmul=True) where the [b, n_ent, K] broadcast would not fit; tests/test_one_vs_all_host.py checks that the two
agree.  Test infrastructure only."""
import numpy as np
import torch

from oracle import ref_step


def query_vectors(model, side, e_s, e_p, e_o):
    """[b, K] rows q with corruption_scores(model, side, ...) = q @ ent.T for DistMult, ComplEx and HolE."""
    K = e_s.shape[1]
    h = K // 2
    if model == "DistMult":
        return e_p * e_o if side == "s" else e_s * e_p
    s_re, s_im, p_re, p_im, o_re, o_im = e_s[:, :h], e_s[:, h:], e_p[:, :h], e_p[:, h:], e_o[:, :h], e_o[:, h:]
    if side == "s":  # ComplEx.py:95-108
        q = torch.cat([p_re * o_re + p_im * o_im, p_re * o_im - p_im * o_re], 1)
    else:  # ComplEx.py:139-150
        q = torch.cat([s_re * p_re - s_im * p_im, s_im * p_re + s_re * p_im], 1)
    return (2.0 / (K / 2.0)) * q if model == "HolE" else q


def side_loss(logits, target, reduction):
    """Per-positive loss over all-entity logits [b, n_ent] (clipped like loss_functions.py:32-35; torch.clamp passes
    the gradient on [-75, 75] only) with the positive's own entity `target` [b]."""
    lc = torch.clamp(logits, ref_step.CLIP_LO, ref_step.CLIP_HI)
    lt = lc.gather(1, target[:, None])[:, 0]
    if reduction == "sum":
        return torch.logsumexp(lc, 1) - lt
    m = lc.max(1, keepdim=True).values.detach()
    ex = torch.exp(lc - m)
    et = ex.gather(1, target[:, None])[:, 0]
    neg_mean = (ex.sum(1) - et) / (lc.shape[1] - 1)  # the reference's reduce over the n_ent - 1 negatives
    return -torch.log(et / (neg_mean + et))


def side_softmax(logits, target, reduction):
    """The row quantities behind side_loss, detached: (lc, P, m, D) with lc the clipped logits [b, n], m each row's
    largest clipped logit, D = w sum_{e != t} exp(lc_e - m) + exp(lc_t - m) (w = 1 for sum, 1 / (n - 1) for mean) and
    P = w_e exp(lc - m) / D (w_t = 1): dL/dl = P - [e == t] where the logit is inside the clip range."""
    lc = torch.clamp(logits.detach(), ref_step.CLIP_LO, ref_step.CLIP_HI)
    m = lc.max(1, keepdim=True).values
    we = torch.full_like(lc, 1.0 if reduction == "sum" else 1.0 / (lc.shape[1] - 1))
    we.scatter_(1, target[:, None], 1.0)
    ex = we * torch.exp(lc - m)
    D = ex.sum(1, keepdim=True)
    return lc, ex / D, m, D


def loss_and_grads(model, ent, rel, triples, sides="s,o", reduction="sum", device="cpu", matmul=False,
                   dtype=torch.float64):
    """(loss, g_ent, g_rel) of one 1vsAll step on dense tables ent [n_ent, K], rel [n_rel, K], in float64 (dtype float32
    evaluates the same graph in fp32)."""
    E = torch.as_tensor(np.asarray(ent), dtype=dtype, device=device).clone().requires_grad_(True)
    R = torch.as_tensor(np.asarray(rel), dtype=dtype, device=device).clone().requires_grad_(True)
    t = torch.as_tensor(np.asarray(triples), dtype=torch.long, device=device)
    e_s, e_p, e_o = E[t[:, 0]], R[t[:, 1]], E[t[:, 2]]
    total = torch.zeros((), dtype=dtype, device=device)
    for side in sides.split(","):
        if matmul:
            logits = query_vectors(model, side, e_s, e_p, e_o) @ E.T
        else:
            logits = ref_step.corruption_scores(model, side, e_s, e_p, e_o, E)
        total = total + side_loss(logits, t[:, 0 if side == "s" else 2], reduction).sum()
    total.backward()
    return float(total.detach()), E.grad.cpu().numpy(), R.grad.cpu().numpy()
