"""fp64 torch model of relation-aware link prediction (Distributed_Sparse::distmultLoss, include/hnh/distmult.hpp) --
TEST INFRASTRUCTURE.

PyG's examples/rgcn_link_pred.py is the definition.  For the stored entries (rows[i], cols[i]) of a target matrix with
relations rels[i] (duplicates count, each under its own relation):
    s    = (H_A[rows] * rel[rels] * H_B[cols]).sum(1)
    loss = F.binary_cross_entropy_with_logits(cat([s_pos, s_neg]), cat([ones, zeros]), reduction="mean")
    correct = #[(s > 0) == (y > 0.5)]
and the gradients by autograd.  An entry whose relation is not an integer in [0, R) contributes nothing (the op's
convention; the targets object refuses such values).  Training is tests/training_oracle.py's step
(torch.optim.AdamW(foreach=False), clip_grad_norm_) over the model's parameters and then rel.  fp64 on the CPU; nothing
under distributed_sddmm_b200/ imports this module.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from tests.rgcn_oracle import valid


def _t(x):
    return torch.as_tensor(np.asarray(x, np.float64))


def _i(x):
    return torch.as_tensor(np.asarray(x, np.int64))


class DistMultDecoder(torch.nn.Module):
    """The decoder of PyG's examples/rgcn_link_pred.py: rel_emb, and (z[src] * rel_emb[edge_type] * z[dst]).sum(-1)."""

    def __init__(self, num_relations, hidden_channels):
        super().__init__()
        self.rel_emb = torch.nn.Parameter(torch.empty(num_relations, hidden_channels, dtype=torch.float64))
        torch.nn.init.xavier_uniform_(self.rel_emb)

    def forward(self, z, edge_index, edge_type):
        z_src, z_dst = z[edge_index[0]], z[edge_index[1]]
        rel = self.rel_emb[edge_type]
        return torch.sum(z_src * rel * z_dst, dim=1)


def scores(H_A, H_B, rel, rows, cols, rels):
    """s per triple (torch tensors in, tensor out); entries that are no relation score 0."""
    ok = torch.as_tensor(valid(rels, rel.shape[0]))
    rho = torch.as_tensor(np.where(ok.numpy(), np.nan_to_num(np.asarray(rels, np.float64)), 0).astype(np.int64))
    s = (H_A[_i(rows)] * rel[rho] * H_B[_i(cols)]).sum(1)
    return torch.where(ok, s, torch.zeros_like(s)), ok


def op(H_A, H_B, rel, rows, cols, rels, target, inv_count, same=False):
    """One distmultLoss call: (loss sum, correct, scores, dH_A, dH_B, drel) as numpy / Python numbers, the loss of
    every valid entry weighted by inv_count for the gradients.  same=True: H_A is H_B, one leaf."""
    a = _t(H_A).clone().requires_grad_()
    b = a if same else _t(H_B).clone().requires_grad_()
    d = _t(rel).clone().requires_grad_()
    s, ok = scores(a, b, d, rows, cols, rels)
    y = torch.full_like(s, float(target))
    terms = F.binary_cross_entropy_with_logits(s, y, reduction="none") * ok
    (terms.sum() * inv_count + (a * 0).sum() + (b * 0).sum() + (d * 0).sum()).backward()
    sd = s.detach()
    correct = int((((sd > 0) == (y > 0.5)) & ok).sum())
    ga = a.grad.numpy().copy()
    return float(terms.detach().sum()), correct, sd.numpy(), ga, ga if same else b.grad.numpy().copy(), d.grad.numpy().copy()


def relational_loss(H, rel, pos, neg):
    """The mean loss of PyG's example over pos = (rows, cols, rels) with target 1 and neg with target 0, from tensors H
    and rel: (loss tensor, correct, count, s_pos, s_neg)."""
    sp, _ = scores(H, H, rel, *pos)
    sn, _ = scores(H, H, rel, *neg)
    s = torch.cat([sp, sn])
    y = torch.cat([torch.ones_like(sp), torch.zeros_like(sn)])
    loss = F.binary_cross_entropy_with_logits(s, y, reduction="mean") if len(s) else (H * 0).sum() + (rel * 0).sum()
    correct = int(((s.detach() > 0) == (y > 0.5)).sum())
    return loss, correct, len(s), sp.detach().numpy(), sn.detach().numpy()


def train(forward, params, rel0, pos, neg, steps, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, max_grad_norm=None):
    """forward(t) -> H from the leaf tensors params.  Trains params and then rel (starting at rel0) for `steps` steps with
    one AdamW; returns (per-step (loss, correct, count, grad_norm), trained rel as numpy)."""
    rel = _t(rel0).clone().requires_grad_()
    leaves = list(params) + [rel]
    opt = torch.optim.AdamW(leaves, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, foreach=False)
    out = []
    for t in range(steps):
        opt.zero_grad()
        loss, correct, count, _, _ = relational_loss(forward(t), rel, pos, neg)
        loss.backward()
        for p in leaves:
            if p.grad is None:
                p.grad = torch.zeros_like(p)
        norm = torch.nn.utils.clip_grad_norm_(leaves, max_grad_norm if max_grad_norm else math.inf)
        out.append((float(loss.detach()), correct, count, float(norm)))
        opt.step()
    return out, rel.detach().numpy().copy()
