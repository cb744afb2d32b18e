"""fp64 models of graph-level prediction (include/hnh/graph_readout.hpp) -- TEST INFRASTRUCTURE.

For node rows H (N x r) and batch[u] the graph of row u (negative: no graph), G graphs:
    sum   P = torch.zeros(G, r).index_add_(0, batch, H)                                 (PyG global_add_pool)
    mean  P = sum / n_g, 0 for an empty graph                                           (PyG global_mean_pool)
    max   P = torch.zeros(G, r).scatter_reduce(0, batch, H, "amax", include_self=False)  (0 for an empty graph)
          with the gradient dP_g,k / C_g,k to each of the C_g,k rows attaining the maximum (Distributed_Sparse::maxAggregate's
          convention; torch's own autograd also counts the untouched zero when the maximum is exactly 0)
    logits = torch.nn.Linear(r, C)(P) with a head (weight = W.T, bias = b), P without
and training is tests/training_oracle.py's step (F.cross_entropy, clip_grad_norm_, torch.optim.AdamW(foreach=False)) over
the model's parameters and then the head's.  The numpy functions give the segment plan and the kernels' results on
their own.  fp64 on the CPU; nothing under distributed_sddmm_b200/ imports this module.
"""
from __future__ import annotations

import numpy as np
import torch

from tests import training_oracle as tro

POOLS = ("sum", "mean", "max")
CHUNK = 256  # HNH_SEGMENT_CHUNK


def _t(x):
    return torch.as_tensor(np.asarray(x, np.float64))


def pool_torch(H, batch, G, pool):
    """P (G x r), differentiable in H, with max's equal split of the gradient over tied rows."""
    batch = np.asarray(batch, np.int64)
    keep = torch.as_tensor(batch >= 0)
    b = torch.as_tensor(batch[batch >= 0])
    h = H[keep]
    r = H.shape[1]
    if pool == "max":
        out = torch.zeros(G, r, dtype=H.dtype).scatter_reduce(0, b[:, None].expand(len(b), r), h, "amax", include_self=False)
        tie = (h == out[b]).detach().to(H.dtype)
        count = torch.zeros(G, r, dtype=H.dtype).index_add(0, b, tie)
        share = torch.zeros(G, r, dtype=H.dtype).index_add(0, b, h * tie / count[b].clamp(min=1))
        return out.detach() + (share - share.detach())
    out = torch.zeros(G, r, dtype=H.dtype).index_add(0, b, h)
    if pool == "mean":
        n = torch.bincount(b, minlength=G).to(H.dtype)
        out = out / n.clamp(min=1)[:, None]
    return out


def head_torch(P, head):
    """torch.nn.Linear(r, C) with weight = W.T and bias = b, as P W + b; head None: P itself."""
    if head is None:
        return P
    W, b = head
    return P @ W + b


def train(forward_H, model_leaves, batch, G, pool, head, labels, steps, **opt):
    """forward_H(t) -> the model's output (N x r) from model_leaves.  Trains model_leaves and the head (W r x C, b C as
    numpy, or None) in place for `steps` steps over the graph labels; returns (per-step results, trained head)."""
    hl = None if head is None else tuple(_t(v).clone().requires_grad_() for v in head)
    res = tro.train(lambda t: head_torch(pool_torch(forward_H(t), batch, G, pool), hl), list(model_leaves) + list(hl or ()),
                    labels, steps, **opt)
    return res, None if hl is None else tuple(v.detach().numpy().copy() for v in hl)


# ---- the segment plan and the kernels in numpy --------------------------------------------------------------------------
def plan(batch, G):
    """(seg_start, seg_rows, chunk_first, chunk_seg) as the library builds them: segment g lists graph g's rows in
    ascending order; every segment is cut into chunks of CHUNK rows, an empty one into one empty chunk."""
    batch = np.asarray(batch, np.int64)
    rows = np.flatnonzero(batch >= 0)
    order = np.argsort(batch[rows], kind="stable")
    seg_rows = rows[order].astype(np.int64)
    counts = np.bincount(batch[rows], minlength=G)
    seg_start = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    nch = np.maximum(1, (counts + CHUNK - 1) // CHUNK)
    chunk_first = np.concatenate([[0], np.cumsum(nch)]).astype(np.int64)
    chunk_seg = np.repeat(np.arange(G), nch).astype(np.int32)
    return seg_start, seg_rows, chunk_first, chunk_seg


def pool_np(H, batch, G, pool):
    """The pool kernel: P (sum; 0 for an empty segment), or (P, C) for max with (-inf, 0) for an empty segment."""
    batch = np.asarray(batch, np.int64)
    sel = batch >= 0
    r = H.shape[1]
    if pool == "max":
        P = np.full((G, r), -np.inf)
        np.maximum.at(P, batch[sel], H[sel])
        C = np.zeros((G, r))
        np.add.at(C, batch[sel], (H[sel] == P[batch[sel]]).astype(np.float64))
        return P, C
    P = np.zeros((G, r))
    np.add.at(P, batch[sel], H[sel])
    return P


def pool_grad_np(batch, G, dP, scale=None, H=None, P=None, C=None):
    """dH_u = scale_g dP_g, or [H_u == P_g] dP_g / C_g with H, P, C; 0 for a row outside [0, G)."""
    batch = np.asarray(batch, np.int64)
    dH = np.zeros((len(batch), dP.shape[1]))
    sel = (batch >= 0) & (batch < G)
    g = batch[sel]
    if H is None:
        dH[sel] = dP[g] * (1.0 if scale is None else np.asarray(scale)[g][:, None])
    else:
        q = np.divide(dP[g], C[g], out=np.zeros_like(dP[g]), where=C[g] != 0)
        dH[sel] = np.where(H[sel] == P[g], q, 0.0)
    return dH
