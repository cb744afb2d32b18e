"""fp64 models of R-GCN with basis decomposition (include/hnh/rgcn.hpp with num_bases) and of basis aggregation
(Distributed_Sparse::basisAggregate) -- TEST INFRASTRUCTURE.

A layer is PyG's RGCNConv(f, r, num_relations=R, num_bases=B, aggr, root_weight=True, bias=True), written out
literally: the relation weights are
    W = (comp @ basis.view(B, -1)).view(R, f, r),   basis = weight.reshape(B, f, r)   (the library's "weight")
and the layer is then tests/rgcn_oracle.py's per-relation model with those weights.  Every gradient comes from torch's
autograd.  The numpy functions give the kernels' sums on their own, in the library's basis-first form:
    H[u, b f + k] = sum_{(u, v) stored} scale[u, rho] comp[rho, b] X[v, k]
    dX[v]         = sum_{(u, v) stored} scale[u, rho] sum_b comp[rho, b] dH[u, b f : b f + f]
    dcomp[rho, b] = sum_{(u, v) stored of relation rho} scale[u, rho] <dH[u, b f : b f + f], X[v]>
fp64 on the CPU; nothing under distributed_sddmm_b200/ imports this module.
"""
from __future__ import annotations

import numpy as np
import torch

from tests import link_prediction_oracle as lpo
from tests import rgcn_oracle as ro
from tests import training_oracle as tro

AGGREGATIONS = ro.AGGREGATIONS
PARAMS = ("weight", "comp", "bias", "root")
_t = ro._t


def relation_weights(P, R, B, f, r):
    """PyG's weight = (comp @ basis.view(B, -1)).view(R, f, r), as the R f x r "weight" of tests/rgcn_oracle.py."""
    return (P["comp"] @ P["weight"].reshape(B, f * r)).reshape(R * f, r)


def model_torch(rows, cols, rels, N, layers, params, X, R, B, aggr):
    """The network output; params[l] = {"weight" (B f x r), "comp" (R x B), "bias", "root"} tensors."""
    merged = [{"weight": relation_weights(P, R, B, f, r), "bias": P["bias"], "root": P["root"]}
              for P, (f, r) in zip(params, layers)]
    return ro.model_torch(rows, cols, rels, N, layers, merged, X, R, aggr)


def random_params(layers, R, B, rng, scale=1.0):
    """Parameters of every layer as numpy dicts, in the library's names."""
    out = []
    for f, r in layers:
        out.append({"weight": rng.uniform(-1, 1, (B * f, r)) * scale / np.sqrt(f), "comp": rng.uniform(-1, 1, (R, B)),
                    "bias": rng.uniform(-0.5, 0.5, r), "root": rng.uniform(-1, 1, (f, r)) * scale / np.sqrt(f)})
    return out


def _leaves(params):
    return [{k: _t(v).clone().requires_grad_() for k, v in P.items()} for P in params]


def forward_backward(rows, cols, rels, N, layers, params, X, R, B, aggr, G):
    """(output, dL/dX, [per-layer dict of dL/d param]) for L = <output, G>, as numpy."""
    tp = _leaves(params)
    x = _t(X).clone().requires_grad_()
    out = model_torch(rows, cols, rels, N, layers, tp, x, R, B, aggr)
    (out * _t(G)).sum().backward()
    grads = [{k: (v.grad if v.grad is not None else torch.zeros_like(v)).numpy().copy() for k, v in P.items()} for P in tp]
    return out.detach().numpy(), x.grad.numpy().copy(), grads


def train(rows, cols, rels, N, layers, params, X, R, B, aggr, labels, steps, **opt):
    """Node classification: trains on the global rows; returns (per-step results, trained params as numpy dicts)."""
    tp = _leaves(params)
    x = _t(X)
    res = tro.train(lambda _: model_torch(rows, cols, rels, N, layers, tp, x, R, B, aggr), [v for P in tp for v in P.values()],
                    labels, steps, **opt)
    return res, [{k: v.detach().numpy().copy() for k, v in P.items()} for P in tp]


def train_link(rows, cols, rels, N, layers, params, X, R, B, aggr, pairs, steps, **opt):
    """Link prediction over pairs = (T rows, T cols, targets); returns as train."""
    tp = _leaves(params)
    x = _t(X)
    res = lpo.link_train_step(pairs)(lambda _: model_torch(rows, cols, rels, N, layers, tp, x, R, B, aggr),
                                     [v for P in tp for v in P.values()], None, steps, **opt)
    return res, [{k: v.detach().numpy().copy() for k, v in P.items()} for P in tp]


# ---- the kernels in numpy ------------------------------------------------------------------------------------------------
def mean_scale(rows, vals, M, R):
    """1 / |N_rho(u)| (M x R), 0 where the count is 0: the model's scale for the mean."""
    c = ro.relation_counts(rows, vals, M, R)
    return np.divide(1.0, c, out=np.zeros_like(c), where=c != 0)


def basis_aggregate(rows, cols, vals, M, X, R, comp, scale=None):
    """H (M x B f)."""
    f, B = X.shape[1], comp.shape[1]
    A = ro.relational_aggregate(rows, cols, vals, M, X, R).reshape(M, R, f)
    if scale is not None:
        A = A * scale[:, :, None]
    return np.einsum("urk,rb->ubk", A, comp).reshape(M, B * f)


def basis_aggregate_backward(rows, cols, vals, dH, X, N, R, comp, scale=None):
    """(dX (N x f), dcomp (R x B))."""
    M, f, B = dH.shape[0], X.shape[1], comp.shape[1]
    dH3 = dH.reshape(M, B, f)
    s = np.ones((M, R)) if scale is None else scale
    dA = np.einsum("rb,ubk->urk", comp, dH3) * s[:, :, None]
    dX = ro.relational_aggregate_backward(rows, cols, vals, dA.reshape(M, R * f), N, R)
    A = ro.relational_aggregate(rows, cols, vals, M, X, R).reshape(M, R, f)
    dcomp = np.einsum("ur,ubk,urk->rb", s, dH3, A)
    return dX, dcomp


def products(rows, cols, vals, dH, X, R, B, scale=None):
    """P (B x nnz): P[b, j] = scale[u, rho] <dH[u, b f : b f + f], X[v]> for entry j = (u, v) of relation rho, 0 for an
    entry that is no relation (u the gathered row, v the stored one of the B order)."""
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    f = X.shape[1]
    ok = ro.valid(vals, R)
    rel = np.where(ok, np.nan_to_num(np.asarray(vals, np.float64)), 0).astype(np.int64)
    w = np.ones(len(rows)) if scale is None else scale[rows, rel]
    P = np.einsum("jbk,jk->bj", dH.reshape(len(dH), B, f)[rows], X[cols]) * w
    P[:, ~ok] = 0.0
    return P
