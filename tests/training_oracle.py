"""fp64 torch model of training (include/hnh/training.hpp) -- TEST INFRASTRUCTURE.

One step is torch's own:
    loss = F.cross_entropy(logits, labels, ignore_index=-1)          (labels < 0 become -1)
    loss.backward(); unread parameters get a zero gradient (as the library's)
    grad_norm = clip_grad_norm_(params, max_grad_norm or inf)         (inf: the norm alone; the coefficient is 1)
    torch.optim.AdamW(params, lr, betas, eps, weight_decay, foreach=False).step()
on the models of tests/graph_transformer_oracle.py, tests/graph_transformer_block_oracle.py and the four GAT oracles.
fp64 on the CPU; nothing under distributed_sddmm_b200/ imports this module.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from tests import gat_additive_oracle as gao
from tests import gat_backward_oracle as gbk
from tests import gat_softmax_oracle as gso
from tests import gatv2_oracle as gv2
from tests import graph_transformer_block_oracle as gbo
from tests import graph_transformer_oracle as gto


def train(forward, params, labels, steps, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, max_grad_norm=None,
          lrs=None):
    """forward(t) -> logits (n x C) from the leaf tensors params.  Trains them in place for `steps` steps and returns
    the per-step (loss, correct, labelled, grad_norm).  lrs: an optional lr per step."""
    opt = torch.optim.AdamW(params, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, foreach=False)
    lab = torch.from_numpy(np.where(np.asarray(labels) < 0, -1, np.asarray(labels)).astype(np.int64))
    m = lab >= 0
    out = []
    for t in range(steps):
        if lrs is not None:
            opt.param_groups[0]["lr"] = lrs[t]
        opt.zero_grad()
        logits = forward(t)
        loss = F.cross_entropy(logits, lab, ignore_index=-1) if m.any() else (logits * 0).sum()
        loss.backward()
        for p in params:
            if p.grad is None:
                p.grad = torch.zeros_like(p)
        norm = torch.nn.utils.clip_grad_norm_(params, max_grad_norm if max_grad_norm else math.inf)
        correct = int((logits.detach().argmax(1)[m] == lab[m]).sum())
        out.append((float(loss.detach()), correct, int(m.sum()), float(norm)))
        opt.step()
    return out


def _leaves(params):
    return [{k: gto._t(v).clone().requires_grad_() for k, v in P.items()} for P in params]


def train_gt(rows, cols, N, layers, params, X, labels, steps, attr=None, beta=False, ffn=0, dropout=0.0, seeds=None, eps=1e-5,
             **opt):
    """Trains a graph transformer (ffn > 0: with blocks) on the global rows; returns (per-step results, trained params
    as numpy dicts).  seeds[t]: the dropout seed of step t."""
    tp = _leaves(params)
    A = gto._t(gto.dense_attributes(rows, cols, N, attr)) if attr is not None else None
    x = gto._t(X)
    seeds = seeds or [0] * steps

    def forward(t):
        if ffn:
            return gbo.model_torch(rows, cols, N, layers, tp, x, A, beta, dropout, seeds[t], eps)
        return gto.model_torch(rows, cols, N, layers, tp, x, A, beta, dropout, seeds[t])

    res = train(forward, [v for P in tp for v in P.values()], labels, steps, **opt)
    return res, [{k: v.detach().numpy().copy() for k, v in P.items()} for P in tp]


def train_gat(kind, rows, cols, N, layers, weights, a1, a2, X, labels, steps, alpha=0.2, **opt):
    """Trains GAT with attention `kind` on the global rows: weights[layer][head], a1 / a2[layer][head].  Returns
    (per-step results, weights, a1, a2) as numpy."""
    ri, ci = gbk.edges(rows, cols, N)
    t = lambda v: torch.tensor(np.asarray(v, np.float64), requires_grad=True)  # noqa: E731
    ws, u1, u2 = [[t(w) for w in l] for l in weights], [[t(v) for v in l] for l in a1], [[t(v) for v in l] for l in a2]
    x = gto._t(X)

    def forward(_):
        if kind == "leaky":
            return gbk.gat_forward_torch(ri, ci, N, layers, ws, alpha, x)
        if kind == "softmax":
            return gso.gat_softmax_forward_torch(ri, ci, N, layers, ws, alpha, x)
        if kind == "additive":
            return gao.gat_additive_forward_torch(ri, ci, N, layers, ws, u1, u2, alpha, x)
        return gv2.gatv2_forward_torch(ri, ci, N, layers, ws, u1, alpha, x)

    params = [w for l in ws for w in l] + [v for l1, l2 in zip(u1, u2) for v in l1 + l2]
    res = train(forward, params, labels, steps, **opt)
    g = lambda nested: [[v.detach().numpy().copy() for v in l] for l in nested]  # noqa: E731
    return res, g(ws), g(u1), g(u2)
