"""fp64 models of GIN / GINE (include/hnh/gin.hpp) and of edge-ReLU aggregation (Distributed_Sparse::edgeReluAggregate)
-- TEST INFRASTRUCTURE.

For the stored entries (rows[i], cols[i]) of S over N nodes (duplicates count; PyG's edge_index = [cols; rows]) and
per-entry attributes attr[i], `layer_torch` is written literally from PyG's GINConv / GINEConv with nn =
Sequential(Linear(f, h), ReLU(), Linear(h, r)):
    m_i = x[cols[i]]                         GINConv's message x_j
    m_i = relu(x[cols[i]] + lin(attr[i]))     GINEConv's message, lin = Linear(edge_dim, f)
    aggr = zeros(N, f).index_add_(0, rows, m)   (the messages materialised, then scattered)
    out  = nn((1 + eps) x + aggr)
and every gradient by torch's autograd.  Training reuses tests/training_oracle.py, tests/link_prediction_oracle.py and
tests/graph_readout_oracle.py.  The numpy functions give edgeReluAggregate and its backward on their own, for the kernel
and multi-rank checks.  fp64 on the CPU; nothing under distributed_sddmm_b200/ imports this module.
"""
from __future__ import annotations

import numpy as np
import torch

from tests import link_prediction_oracle as lpo
from tests import training_oracle as tro


def _t(x):
    return torch.as_tensor(np.asarray(x, np.float64))


def attr_of(rows, cols, e):
    """Edge attributes as a function of the global S-row and S-column only (stored duplicates share them)."""
    rows, cols = np.asarray(rows, np.float64), np.asarray(cols, np.float64)
    return np.cos(0.31 * rows[:, None] + 0.73 * cols[:, None] + 0.45 * np.arange(e)[None, :])


def edge_rows(rows, cols, f):
    """Integer-valued f-wide per-entry rows as a function of the global (u, v) only (duplicates share them); with integer
    X, X_v + E_i == 0 happens, which the strict mask must see."""
    rows, cols = np.asarray(rows, np.float64), np.asarray(cols, np.float64)
    return np.round(3.0 * np.cos(0.37 * rows[:, None] + 0.91 * cols[:, None] + 0.53 * np.arange(f)[None, :]))


def layer_torch(rows, cols, N, x, P, attr=None):
    """One GINConv (attr None) or GINEConv layer; P = {"lin1", "lin1_bias", "lin2", "lin2_bias", "eps"[, "edge",
    "edge_bias"]} tensors, weights input-major."""
    ri, ci = torch.as_tensor(np.asarray(rows, np.int64)), torch.as_tensor(np.asarray(cols, np.int64))
    msg = x[ci]
    if attr is not None:
        msg = torch.relu(msg + (attr @ P["edge"] + P["edge_bias"]))
    aggr = torch.zeros(N, x.shape[1], dtype=x.dtype).index_add_(0, ri, msg)
    h = aggr + (1 + P["eps"]) * x
    return torch.relu(h @ P["lin1"] + P["lin1_bias"]) @ P["lin2"] + P["lin2_bias"]


def model_torch(rows, cols, N, layers, params, X, attr=None):
    """The network output: every layer but the last ends in a ReLU; attr (nnz x edge_dim tensor) makes it GINE."""
    h = X
    for l, P in enumerate(params):
        y = layer_torch(rows, cols, N, h, P, attr)
        h = torch.relu(y) if l + 1 < len(layers) else y
    return h


def random_params(layers, edge_dim, rng, eps=0.25, scale=1.0):
    """Parameters of every layer as numpy dicts, in the library's names."""
    out = []
    for f, h, r in layers:
        P = {"lin1": rng.uniform(-1, 1, (f, h)) * scale / np.sqrt(f), "lin1_bias": rng.uniform(-0.5, 0.5, h),
             "lin2": rng.uniform(-1, 1, (h, r)) * scale / np.sqrt(h), "lin2_bias": rng.uniform(-0.5, 0.5, r)}
        if edge_dim:
            P["edge"] = rng.uniform(-1, 1, (edge_dim, f)) / np.sqrt(edge_dim)
            P["edge_bias"] = rng.uniform(-0.5, 0.5, f)
        P["eps"] = np.array([eps + 0.1 * len(out)])
        out.append(P)
    return out


def _leaves(params, train_eps=True):
    """Tensors of every layer: leaves with gradients, eps a constant unless train_eps."""
    return [{k: _t(v).clone().requires_grad_(train_eps or k != "eps") for k, v in P.items()} for P in params]


def _trained(tp):
    return [v for P in tp for v in P.values() if v.requires_grad]


def forward_backward(rows, cols, N, layers, params, X, G, attr=None):
    """(output, dL/dX, [per-layer dict of dL/d param]) for L = <output, G>, as numpy."""
    tp = _leaves(params)
    x = _t(X).clone().requires_grad_()
    out = model_torch(rows, cols, N, layers, tp, x, None if attr is None else _t(attr))
    (out * _t(G)).sum().backward()
    grads = [{k: v.grad.numpy().copy() for k, v in P.items()} for P in tp]
    return out.detach().numpy(), x.grad.numpy().copy(), grads


def train(rows, cols, N, layers, params, X, labels, steps, attr=None, train_eps=True, **opt):
    """Node classification on the global rows; returns (per-step results, trained params as numpy dicts)."""
    tp = _leaves(params, train_eps)
    x, a = _t(X), None if attr is None else _t(attr)
    res = tro.train(lambda _: model_torch(rows, cols, N, layers, tp, x, a), _trained(tp), labels, steps, **opt)
    return res, [{k: v.detach().numpy().copy() for k, v in P.items()} for P in tp]


def train_link(rows, cols, N, layers, params, X, pairs, steps, attr=None, train_eps=True, **opt):
    """Link prediction over pairs = (T rows, T cols, targets); returns as train."""
    tp = _leaves(params, train_eps)
    x, a = _t(X), None if attr is None else _t(attr)
    res = lpo.link_train_step(pairs)(lambda _: model_torch(rows, cols, N, layers, tp, x, a), _trained(tp), None, steps, **opt)
    return res, [{k: v.detach().numpy().copy() for k, v in P.items()} for P in tp]


# ---- edge-ReLU aggregation in numpy ------------------------------------------------------------------------------------
def edge_relu_aggregate(rows, cols, M, X, E):
    """A[u] = sum over the entries i = (u, v) of relu(X[v] + E[i]) (M rows; 0 on an empty row)."""
    A = np.zeros((M, X.shape[1]))
    np.add.at(A, np.asarray(rows, np.int64), np.maximum(X[np.asarray(cols, np.int64)] + E, 0.0))
    return A


def edge_relu_aggregate_backward(rows, cols, X, E, dA, N):
    """(dX, dE): dE[i] = [X[v] + E[i] > 0] dA[u] (the strict mask), dX[v] = the sum of dE[i] over the entries of v."""
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    dE = np.where(X[cols] + E > 0, dA[rows], 0.0)
    dX = np.zeros((N, X.shape[1]))
    np.add.at(dX, cols, dE)
    return dX, dE
