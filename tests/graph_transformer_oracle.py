"""fp64 model of the graph transformer (include/hnh/graph_transformer.hpp) -- TEST INFRASTRUCTURE.

Written from the formulas on a dense masked score matrix, independently of the sparse-attention oracles.  Per layer
with input X, H heads of width d and r = H d:
    Q, K, V, R = X W_q + b_q, X W_k + b_k, X W_v + b_v, X W_s + b_s,   E[u, v] = attr[u, v] W_e  (edge_dim > 0)
    x[u, v, h] = <Q_u,h, K_v,h + E_uv,h> / sqrt(d) + log count(u, v)   where S stores (u, v) count(u, v) > 0 times,
    alpha = the softmax of x over v (rows without entries: 0),  M_u,h = sum_v D_uv,h / (1 - p) alpha (V_v,h + E_uv,h)
    Y = M + R, or with the gate beta_u = sigmoid(w_beta . [M_u, R_u, M_u - R_u]), Y = beta R + (1 - beta) M
    X_next = ReLU(Y), except after the last layer
with D the keep bits of tests/sparse_attention_dropout_oracle.py at seed + the heads of the earlier layers + h.
Duplicate stored pairs are the log count term: each copy contributes exp(x) to the row's sum and its value once.
fp64 on the CPU; nothing under distributed_sddmm_b200/ imports this module.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from tests import sparse_attention_dropout_oracle as sd

PROJECTIONS = ("query", "key", "value", "skip")


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x, np.float64))


def random_params(layers, edge_dim, beta, rng, scale=0.4):
    """Per layer a dict name -> numpy array in the library's layout (weights input-major)."""
    out = []
    for f, d, H in layers:
        r = d * H
        p = {}
        for name in PROJECTIONS:
            p[name] = rng.uniform(-scale, scale, (f, r)) / math.sqrt(f)
            p[name + "_bias"] = rng.uniform(-scale, scale, r)
        if edge_dim:
            p["edge"] = rng.uniform(-scale, scale, (edge_dim, r)) / math.sqrt(edge_dim)
        if beta:
            p["beta"] = rng.uniform(-1, 1, 3 * r)
        out.append(p)
    return out


def dense_attributes(rows, cols, N, attr):
    """The per-entry attributes (nnz x e) as an N x N x e array (stored duplicates of (u, v) share one row)."""
    A = np.zeros((N, N, attr.shape[1]))
    A[rows, cols] = attr
    return A


def keep_weights(rows, cols, N, layers, p, seed):
    """Per layer an H x N x N array of D / (1 - p) at the stored pairs (ones without dropout)."""
    out = []
    s = seed
    for _, _, H in layers:
        W = np.ones((H, N, N))
        if p > 0:
            W[:, rows, cols] = sd.weights(rows, cols, H, p, s).T
        out.append(W)
        s += H
    return out


def model_torch(rows, cols, N, layers, params, X, attr=None, beta=False, p=0.0, seed=0):
    """Output of the network (N x r_last) as a torch tensor.  params: per layer a dict name -> tensor; attr: an
    N x N x e tensor (dense_attributes) or None."""
    count = np.zeros((N, N))
    np.add.at(count, (rows, cols), 1.0)
    mask = torch.from_numpy(count > 0)
    logc = torch.from_numpy(np.log(np.where(count > 0, count, 1.0)))
    has = mask.any(1)
    keep = [torch.from_numpy(w) for w in keep_weights(rows, cols, N, layers, p, seed)]
    for l, (f, d, H) in enumerate(layers):
        P = params[l]
        Q, K, V, R = (X @ P[n] + P[n + "_bias"] for n in PROJECTIONS)
        E = attr @ P["edge"] if attr is not None else None
        Ms = []
        for h in range(H):
            w = slice(h * d, (h + 1) * d)
            Kh = K[None, :, w] + E[:, :, w] if E is not None else K[None, :, w].expand(N, N, d)
            Vh = V[None, :, w] + E[:, :, w] if E is not None else V[None, :, w].expand(N, N, d)
            x = torch.einsum("ud,uvd->uv", Q[:, w], Kh) / math.sqrt(d) + logc
            x = torch.where(mask, x, torch.full_like(x, -torch.inf))
            x = torch.where(has[:, None], x, torch.zeros_like(x))  # rows without entries: any finite row, zeroed below
            a = torch.softmax(x, 1) * has[:, None] * keep[l][h]
            Ms.append(torch.einsum("uv,uvd->ud", a, Vh))
        M = torch.cat(Ms, 1)
        if beta:
            b = torch.sigmoid(torch.cat([M, R, M - R], 1) @ P["beta"])[:, None]
            Y = b * R + (1 - b) * M
        else:
            Y = M + R
        X = torch.relu(Y) if l + 1 < len(layers) else Y
    return X


def forward_np(rows, cols, N, layers, params, X, attr=None, beta=False, p=0.0, seed=0):
    """The network output as numpy; attr: per-entry attributes (nnz x e) or None."""
    A = _t(dense_attributes(rows, cols, N, attr)) if attr is not None else None
    with torch.no_grad():
        return model_torch(rows, cols, N, layers, [{k: _t(v) for k, v in P.items()} for P in params], _t(X), A, beta, p,
                           seed).numpy()


def backward_np(rows, cols, N, layers, params, X, G, attr=None, beta=False, p=0.0, seed=0):
    """(dX, [per layer dict name -> gradient]) of <G, output> as numpy."""
    A = _t(dense_attributes(rows, cols, N, attr)) if attr is not None else None
    tp = [{k: _t(v).requires_grad_() for k, v in P.items()} for P in params]
    x = _t(X).requires_grad_()
    out = model_torch(rows, cols, N, layers, tp, x, A, beta, p, seed)
    out.backward(_t(G))
    return x.grad.numpy(), [{k: v.grad.numpy() for k, v in P.items()} for P in tp]
