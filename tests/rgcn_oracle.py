"""fp64 models of R-GCN (include/hnh/rgcn.hpp) and of relational aggregation (Distributed_Sparse::relationalAggregate)
-- TEST INFRASTRUCTURE.

For the stored entries (rows[i], cols[i]) of S over N nodes with relations rels[i] (duplicates count, each under its
own relation) and a layer of input width f:
    A_rho = torch.zeros(N, f).scatter_reduce(0, rows[rels == rho], X[cols[rels == rho]], "mean" | "sum",
                                             include_self=False)          (0 where a row has no entry of relation rho)
    Y = sum_rho A_rho @ W[rho] + X @ root + bias,   W = weight.reshape(R, f, r)  (PyG's RGCNConv without decomposition)
    X_{l+1} = ReLU(Y) except after the last layer
and every gradient by torch's autograd.  An entry whose relation is not an integer in [0, R) belongs to no relation.
Training reuses tests/training_oracle.py's step (torch.optim.AdamW(foreach=False), clip_grad_norm_) and
tests/link_prediction_oracle.py's link loss.  The numpy functions give the two kernels' sums on their own, for the
kernel and multi-rank checks.  fp64 on the CPU; nothing under distributed_sddmm_b200/ imports this module.
"""
from __future__ import annotations

import numpy as np
import torch

from tests import link_prediction_oracle as lpo
from tests import training_oracle as tro

AGGREGATIONS = ("mean", "sum")
PARAMS = ("weight", "bias", "root")


def _t(x):
    return torch.as_tensor(np.asarray(x, np.float64))


def model_torch(rows, cols, rels, N, layers, params, X, R, aggr):
    """The network output; params[l] = {"weight", "bias", "root"} tensors (R f x r, r, f x r)."""
    rows = torch.as_tensor(np.asarray(rows, np.int64))
    cols = torch.as_tensor(np.asarray(cols, np.int64))
    rels = np.asarray(rels, np.float64)
    h = X
    for l, P in enumerate(params):
        f, r = layers[l]
        W = P["weight"].reshape(R, f, r)
        y = h @ P["root"] + P["bias"]
        for rho in range(R):
            sel = torch.as_tensor(rels == rho)
            ru, cv = rows[sel], cols[sel]
            A = torch.zeros(N, f, dtype=h.dtype).scatter_reduce(0, ru[:, None].expand(len(ru), f), h[cv], aggr,
                                                                include_self=False)
            y = y + A @ W[rho]
        h = torch.relu(y) if l + 1 < len(layers) else y
    return h


def random_params(layers, R, rng, scale=1.0):
    """Parameters of every layer as numpy dicts, in the library's names."""
    out = []
    for f, r in layers:
        out.append({"weight": rng.uniform(-1, 1, (R * f, r)) * scale / np.sqrt(f), "bias": rng.uniform(-0.5, 0.5, r),
                    "root": rng.uniform(-1, 1, (f, r)) * scale / np.sqrt(f)})
    return out


def _leaves(params):
    return [{k: _t(v).clone().requires_grad_() for k, v in P.items()} for P in params]


def forward_backward(rows, cols, rels, N, layers, params, X, R, aggr, G):
    """(output, dL/dX, [per-layer dict of dL/d param]) for L = <output, G>, as numpy."""
    tp = _leaves(params)
    x = _t(X).clone().requires_grad_()
    out = model_torch(rows, cols, rels, N, layers, tp, x, R, aggr)
    (out * _t(G)).sum().backward()
    grads = [{k: (v.grad if v.grad is not None else torch.zeros_like(v)).numpy().copy() for k, v in P.items()} for P in tp]
    return out.detach().numpy(), x.grad.numpy().copy(), grads


def train(rows, cols, rels, N, layers, params, X, R, aggr, labels, steps, **opt):
    """Node classification: trains on the global rows; returns (per-step results, trained params as numpy dicts)."""
    tp = _leaves(params)
    x = _t(X)
    res = tro.train(lambda _: model_torch(rows, cols, rels, N, layers, tp, x, R, aggr), [v for P in tp for v in P.values()],
                    labels, steps, **opt)
    return res, [{k: v.detach().numpy().copy() for k, v in P.items()} for P in tp]


def train_link(rows, cols, rels, N, layers, params, X, R, aggr, pairs, steps, **opt):
    """Link prediction over pairs = (T rows, T cols, targets); returns as train."""
    tp = _leaves(params)
    x = _t(X)
    res = lpo.link_train_step(pairs)(lambda _: model_torch(rows, cols, rels, N, layers, tp, x, R, aggr),
                                     [v for P in tp for v in P.values()], None, steps, **opt)
    return res, [{k: v.detach().numpy().copy() for k, v in P.items()} for P in tp]


# ---- the kernels in numpy ------------------------------------------------------------------------------------------------
def valid(vals, R):
    """Which stored values are relations: integers in [0, R) (NaN, infinities and fractions are not)."""
    v = np.asarray(vals, np.float64)
    with np.errstate(invalid="ignore"):
        return (v >= 0) & (v < R) & (np.floor(v) == v)


def relational_aggregate(rows, cols, vals, M, X, R):
    """A (M x R f): A[u, rho f + k] = sum of X[v, k] over the stored (u, v) of relation rho."""
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    ok = valid(vals, R)
    rel = np.where(ok, np.nan_to_num(np.asarray(vals, np.float64)), 0).astype(np.int64)
    f = X.shape[1]
    A = np.zeros((M, R, f))
    np.add.at(A, (rows[ok], rel[ok]), X[cols[ok]])
    return A.reshape(M, R * f)


def relation_counts(rows, vals, M, R):
    """|N_rho(u)| (M x R)."""
    return relational_aggregate(rows, np.zeros(len(rows), np.int64), vals, M, np.ones((1, 1)), R)


def relational_aggregate_backward(rows, cols, vals, dA, N, R):
    """dX (N x f): dX[v] = sum of dA[u, rho f : rho f + f] over the stored (u, v), rho their relation."""
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    ok = valid(vals, R)
    rel = np.where(ok, np.nan_to_num(np.asarray(vals, np.float64)), 0).astype(np.int64)
    f = dA.shape[1] // R
    dX = np.zeros((N, f))
    np.add.at(dX, cols[ok], dA.reshape(len(dA), R, f)[rows[ok], rel[ok]])
    return dX


def hashed_relations(rows, cols, N, R):
    """A relation for every tuple hashed from (u, v, copy), copy counting the earlier copies of the pair in the list, so
    that duplicates of a pair carry different relations."""
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    keys = rows * N + cols
    o = np.argsort(keys, kind="stable")
    ks = keys[o]
    start = np.r_[0, np.flatnonzero(ks[1:] != ks[:-1]) + 1]
    copy = np.empty(len(ks), np.int64)
    copy[o] = np.arange(len(ks)) - np.repeat(start, np.diff(np.r_[start, len(ks)]))
    return ((rows * 31 + cols * 17 + copy * 7) % R).astype(np.float64)
