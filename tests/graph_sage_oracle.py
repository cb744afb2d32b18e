"""fp64 models of GraphSAGE (include/hnh/graph_sage.hpp) and of max aggregation (Distributed_Sparse::maxAggregate) --
TEST INFRASTRUCTURE.

For the stored entries (rows[i], cols[i]) of S over N nodes (duplicates count) and a layer of input width f:
    A = aggr(X)     torch.zeros(N, f).scatter_reduce(0, rows, X[cols], "sum" | "mean" | "amax", include_self=False)
                    (a row without entries stays 0), PyG's SumAggregation / MeanAggregation / MaxAggregation
    Y = A W_l + b_l + X W_r,   X_{l+1} = ReLU(Y) except after the last layer
and every gradient by torch's autograd; the C entries that attain a maximum share its gradient equally (dZ / C).  Training reuses
tests/training_oracle.py's step (torch.optim.AdamW(foreach=False), clip_grad_norm_) and
tests/link_prediction_oracle.py's link loss.  The numpy functions give max aggregation and its backward on their own,
for the kernel and multi-rank checks.  fp64 on the CPU; nothing under distributed_sddmm_b200/ imports this module.
"""
from __future__ import annotations

import numpy as np
import torch

from tests import link_prediction_oracle as lpo
from tests import training_oracle as tro

AGGREGATIONS = ("mean", "sum", "max")
_REDUCE = {"mean": "mean", "sum": "sum", "max": "amax"}


def _t(x):
    return torch.as_tensor(np.asarray(x, np.float64))


def aggregate_torch(rows, cols, N, X, aggr):
    """aggr(X) (torch, differentiable in X) over the stored entries (rows[i], cols[i]).  For "max" the value is
    scatter_reduce's and the gradient dZ_u / C_u goes to each of the C_u entries attaining the maximum.  (torch's own
    autograd of scatter_reduce(include_self=False) also counts the untouched zero of `self` as a tie when the maximum is
    exactly 0, and so gives each attaining entry dZ_u / (C_u + 1) there; tests/test_graph_sage.py shows both.)"""
    rows = torch.as_tensor(np.asarray(rows, np.int64))
    cols = torch.as_tensor(np.asarray(cols, np.int64))
    f = X.shape[1]
    index = rows[:, None].expand(len(rows), f)
    out = torch.zeros(N, f, dtype=X.dtype).scatter_reduce(0, index, X[cols], _REDUCE[aggr], include_self=False)
    if aggr != "max":
        return out
    tie = (X[cols] == out[rows]).detach().to(X.dtype)
    count = torch.zeros(N, f, dtype=X.dtype).index_add(0, rows, tie)
    share = torch.zeros(N, f, dtype=X.dtype).index_add(0, rows, X[cols] * tie / count[rows].clamp(min=1))
    return out.detach() + (share - share.detach())


def model_torch(rows, cols, N, layers, params, X, aggr):
    """The network output; params[l] = {"neigh", "neigh_bias", "root"} tensors (f x r, r, f x r)."""
    h = X
    for l, P in enumerate(params):
        y = aggregate_torch(rows, cols, N, h, aggr) @ P["neigh"] + P["neigh_bias"] + h @ P["root"]
        h = torch.relu(y) if l + 1 < len(layers) else y
    return h


def random_params(layers, rng, scale=1.0):
    """Parameters of every layer as numpy dicts, in the library's names."""
    out = []
    for f, r in layers:
        out.append({"neigh": rng.uniform(-1, 1, (f, r)) * scale / np.sqrt(f), "neigh_bias": rng.uniform(-0.5, 0.5, r),
                    "root": rng.uniform(-1, 1, (f, r)) * scale / np.sqrt(f)})
    return out


def forward_backward(rows, cols, N, layers, params, X, aggr, G):
    """(output, dL/dX, [per-layer dict of dL/d param]) for L = <output, G>, as numpy."""
    tp = [{k: _t(v).clone().requires_grad_() for k, v in P.items()} for P in params]
    x = _t(X).clone().requires_grad_()
    out = model_torch(rows, cols, N, layers, tp, x, aggr)
    (out * _t(G)).sum().backward()
    grads = [{k: (v.grad if v.grad is not None else torch.zeros_like(v)).numpy().copy() for k, v in P.items()} for P in tp]
    return out.detach().numpy(), x.grad.numpy().copy(), grads


def _leaves(params):
    return [{k: _t(v).clone().requires_grad_() for k, v in P.items()} for P in params]


def train(rows, cols, N, layers, params, X, aggr, labels, steps, **opt):
    """Node classification: trains on the global rows; returns (per-step results, trained params as numpy dicts)."""
    tp = _leaves(params)
    x = _t(X)
    res = tro.train(lambda _: model_torch(rows, cols, N, layers, tp, x, aggr), [v for P in tp for v in P.values()], labels,
                    steps, **opt)
    return res, [{k: v.detach().numpy().copy() for k, v in P.items()} for P in tp]


def train_link(rows, cols, N, layers, params, X, aggr, pairs, steps, **opt):
    """Link prediction over pairs = (T rows, T cols, targets); returns as train."""
    tp = _leaves(params)
    x = _t(X)
    res = lpo.link_train_step(pairs)(lambda _: model_torch(rows, cols, N, layers, tp, x, aggr),
                                     [v for P in tp for v in P.values()], None, steps, **opt)
    return res, [{k: v.detach().numpy().copy() for k, v in P.items()} for P in tp]


# ---- max aggregation in numpy ------------------------------------------------------------------------------------------
def max_aggregate(rows, cols, M, X):
    """(Z, C): Z[u] = the column-wise max of X[v] over the stored (u, v), C[u] the number of entries attaining it; both 0
    on a row without entries."""
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    f = X.shape[1]
    Z = np.full((M, f), -np.inf)
    np.maximum.at(Z, rows, X[cols])
    C = np.zeros((M, f))
    np.add.at(C, rows, (X[cols] == Z[rows]).astype(np.float64))
    Z[C == 0] = 0.0
    return Z, C


def max_aggregate_backward(rows, cols, Z, C, dZ, N, X):
    """dX[v] = sum over the stored (u, v) of [X[v] == Z[u]] dZ[u] / C[u] (N rows)."""
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    G = np.divide(dZ, C, out=np.zeros_like(dZ), where=C != 0)
    dX = np.zeros((N, X.shape[1]))
    np.add.at(dX, cols, np.where(X[cols] == Z[rows], G[rows], 0.0))
    return dX
