"""fp64 model of the graph transformer with transformer blocks (GraphTransformer with ffn_ratio > 0) -- TEST
INFRASTRUCTURE.

Every layer is the TransformerConv of tests/graph_transformer_oracle.py without its ReLU (Y), followed by
    H1 = layer_norm(Y; norm1, norm1_bias, eps),  A = H1 W1 + b1,  F = ReLU(A) W2 + b2,
    X_next = layer_norm(H1 + F; norm2, norm2_bias, eps)
with [W1; b1] = ffn1 ((r + 1) x h) and [W2; b2] = ffn2 ((h + 1) x r), in the library's input-major layout.  Layer l
draws its dropout masks at seed + the heads of the earlier layers, as the library does.  fp64 on the CPU; nothing
under distributed_sddmm_b200/ imports this module.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from tests import graph_transformer_oracle as gto

BLOCK = ("norm1", "norm1_bias", "ffn1", "ffn2", "norm2", "norm2_bias")


def random_params(layers, edge_dim, beta, ffn_ratio, rng, scale=0.4):
    """gto.random_params plus, with ffn_ratio > 0, the block's parameters of every layer (LayerNorm gains near 1)."""
    out = gto.random_params(layers, edge_dim, beta, rng, scale)
    for (f, d, H), p in zip(layers, out if ffn_ratio > 0 else []):
        r = d * H
        h = ffn_ratio * r
        for n in ("norm1", "norm2"):
            p[n] = 1 + rng.uniform(-scale, scale, r)
            p[n + "_bias"] = rng.uniform(-scale, scale, r)
        p["ffn1"] = rng.uniform(-1, 1, (r + 1, h)) / math.sqrt(r)
        p["ffn2"] = rng.uniform(-1, 1, (h + 1, r)) / math.sqrt(h)
    return out


def block(Y, P, eps):
    """The block on a layer's TransformerConv output Y (torch)."""
    r = Y.shape[1]
    h1 = F.layer_norm(Y, (r,), P["norm1"], P["norm1_bias"], eps)
    a = h1 @ P["ffn1"][:-1] + P["ffn1"][-1]
    f = torch.relu(a) @ P["ffn2"][:-1] + P["ffn2"][-1]
    return F.layer_norm(h1 + f, (r,), P["norm2"], P["norm2_bias"], eps)


def model_torch(rows, cols, N, layers, params, X, attr=None, beta=False, p=0.0, seed=0, eps=1e-5):
    """Output of the network (N x r_last) as a torch tensor; arguments as gto.model_torch."""
    s = seed
    for l, lay in enumerate(layers):
        Y = gto.model_torch(rows, cols, N, [lay], [params[l]], X, attr, beta, p, s)  # one layer: no ReLU
        X = block(Y, params[l], eps)
        s += lay[2]
    return X


def forward_np(rows, cols, N, layers, params, X, attr=None, beta=False, p=0.0, seed=0, eps=1e-5):
    A = gto._t(gto.dense_attributes(rows, cols, N, attr)) if attr is not None else None
    with torch.no_grad():
        return model_torch(rows, cols, N, layers, [{k: gto._t(v) for k, v in P.items()} for P in params], gto._t(X), A, beta,
                           p, seed, eps).numpy()


def backward_np(rows, cols, N, layers, params, X, G, attr=None, beta=False, p=0.0, seed=0, eps=1e-5):
    """(dX, [per layer dict name -> gradient]) of <G, output> as numpy."""
    A = gto._t(gto.dense_attributes(rows, cols, N, attr)) if attr is not None else None
    tp = [{k: gto._t(v).requires_grad_() for k, v in P.items()} for P in params]
    x = gto._t(X).requires_grad_()
    out = model_torch(rows, cols, N, layers, tp, x, A, beta, p, seed, eps)
    out.backward(gto._t(G))
    return x.grad.numpy(), [{k: v.grad.numpy() for k, v in P.items()} for P in tp]
