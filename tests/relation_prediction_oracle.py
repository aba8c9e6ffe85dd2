"""Float64 oracle of the relation-prediction term of 1vsAll training (kge_one_vs_all_relation_step, DESIGN.md 3.14):
lambda * the multiclass NLL of every positive's relation against every relation, scored as f(s, r, o), alone or added to
the entity sides of tests/one_vs_all_oracle.py, with the gradients of both tables from torch autograd.  The all-relation
logits are Qp(s, o) @ rel.T (matmul=True) or oracle.ref_step.compute_scores on every (s, r, o) (the broadcast form);
tests/test_relation_prediction_host.py checks that the two agree.  Test infrastructure only."""
import numpy as np
import torch

import one_vs_all_oracle
from oracle import ref_step


def relation_query(model, e_s, e_o):
    """[b, K] rows Qp = d f(s, p, o) / dp, so that f(s, r, o) = <x_r, Qp> for DistMult, ComplEx and HolE."""
    K = e_s.shape[1]
    if model == "DistMult":
        return e_s * e_o
    h = K // 2
    s_re, s_im, o_re, o_im = e_s[:, :h], e_s[:, h:], e_o[:, :h], e_o[:, h:]
    q = torch.cat([s_re * o_re + s_im * o_im, s_re * o_im - s_im * o_re], 1)
    return (2.0 / (K / 2.0)) * q if model == "HolE" else q


def relation_logits(model, e_s, e_o, R, matmul=False):
    """[b, n_rel] logits f(s_b, r, o_b) of every relation r."""
    if matmul:
        return relation_query(model, e_s, e_o) @ R.T
    b, n_rel = e_s.shape[0], R.shape[0]
    rep = lambda x: x.repeat_interleave(n_rel, 0)
    return ref_step.compute_scores(model, rep(e_s), R.repeat(b, 1), rep(e_o)).view(b, n_rel)


def loss_and_grads(model, ent, rel, triples, weight=1.0, reduction="sum", sides=None, device="cpu", matmul=False,
                   dtype=torch.float64):
    """(loss, g_ent, g_rel) of weight * L_p, plus L_s + L_o of one_vs_all_oracle on `sides` ('s,o', 'o', 's' or None
    for the relation term alone), on dense tables ent [n_ent, K], rel [n_rel, K]; in float64 (dtype float32 evaluates
    the same graph in fp32)."""
    E = torch.as_tensor(np.asarray(ent), dtype=dtype, device=device).clone().requires_grad_(True)
    R = torch.as_tensor(np.asarray(rel), dtype=dtype, device=device).clone().requires_grad_(True)
    t = torch.as_tensor(np.asarray(triples), dtype=torch.long, device=device)
    e_s, e_p, e_o = E[t[:, 0]], R[t[:, 1]], E[t[:, 2]]
    total = weight * one_vs_all_oracle.side_loss(relation_logits(model, e_s, e_o, R, matmul), t[:, 1], reduction).sum()
    for side in (sides.split(",") if sides else ()):
        if matmul:
            logits = one_vs_all_oracle.query_vectors(model, side, e_s, e_p, e_o) @ E.T
        else:
            logits = ref_step.corruption_scores(model, side, e_s, e_p, e_o, E)
        total = total + one_vs_all_oracle.side_loss(logits, t[:, 0 if side == "s" else 2], reduction).sum()
    total.backward()
    return float(total.detach()), E.grad.cpu().numpy(), R.grad.cpu().numpy()
