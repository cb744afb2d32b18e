"""Autograd model of softmax graph attention -- TEST INFRASTRUCTURE.

The model of tests/gat_backward_oracle.py with the attention normalised over each node's neighbours:
alpha_u. = softmax over the stored entries of row u of S of leaky_relu(e_u.).  The row maximum that keeps exp finite
comes from scatter_reduce(..., "amax") and is detached (the softmax does not depend on it).  fp64 on the CPU, as the
leaky model; nothing under distributed_sddmm_b200/ imports this module.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from tests.gat_backward_oracle import edges


def edge_softmax_torch(x, ri, N):
    """Softmax of the edge values x over each row: ri[k] is the row of edge k (rows without edges are unused)."""
    m = torch.full((N,), -torch.inf, dtype=x.dtype).scatter_reduce(0, ri, x.detach(), "amax", include_self=True)
    ex = torch.exp(x - m[ri])
    s = torch.zeros(N, dtype=x.dtype).index_add(0, ri, ex)
    return ex / s[ri]


def gat_softmax_forward_torch(ri, ci, N, layers, weights, alpha, X0):
    """Per head: H = X W; e_uv = <H_u, H_v> on every stored (u, v); a = edge_softmax(leaky_relu(e)); Z = S_a H; the
    head's output window = relu(Z)."""
    X = X0
    for (fin, fph, heads), ws in zip(layers, weights):
        outs = []
        for h in range(heads):
            H = X @ ws[h]
            e = (H[ri] * H[ci]).sum(1)
            a = edge_softmax_torch(F.leaky_relu(e, alpha), ri, N)
            Z = torch.zeros(N, fph, dtype=H.dtype).index_add(0, ri, a[:, None] * H[ci])
            outs.append(torch.relu(Z))
        X = torch.cat(outs, 1)
    return X


def gat_softmax_backward_global(rows, cols, N, layers, weights, alpha, X0, grad_out):
    """Gradients of <grad_out, GAT_softmax(X0)> (global matrices): (dX0, dW[layer][head]) as numpy arrays."""
    ri, ci = edges(rows, cols, N)
    x = torch.tensor(np.asarray(X0, np.float64), requires_grad=True)
    ws = [[torch.tensor(np.asarray(w, np.float64), requires_grad=True) for w in per_layer] for per_layer in weights]
    out = gat_softmax_forward_torch(ri, ci, N, layers, ws, alpha, x)
    out.backward(torch.from_numpy(np.asarray(grad_out, np.float64)))
    return x.grad.numpy(), [[w.grad.numpy() for w in per_layer] for per_layer in ws]


def gat_softmax_forward_global(rows, cols, N, layers, weights, alpha, X0):
    """The forward pass of the model above, as numpy."""
    ri, ci = edges(rows, cols, N)
    with torch.no_grad():
        ws = [[torch.from_numpy(np.asarray(w, np.float64)) for w in per_layer] for per_layer in weights]
        return gat_softmax_forward_torch(ri, ci, N, layers, ws, alpha, torch.from_numpy(np.asarray(X0, np.float64))).numpy()


def edge_softmax_np(x, r, N):
    """numpy edge softmax per row (the reference the library's edgeSoftmax is checked against); x, r: 1-D."""
    x = np.asarray(x, np.float64)
    m = np.full(N, -np.inf)
    np.maximum.at(m, r, x)
    ex = np.exp(x - m[r])
    s = np.zeros(N)
    np.add.at(s, r, ex)
    return ex / s[r]


def edge_softmax_backward_np(a, g, r, N):
    """numpy backward of the edge softmax: a = its output, g = dL/da; returns dL/dx = a (g - t), t_u = sum_u a g."""
    t = np.zeros(N)
    np.add.at(t, r, a * g)
    return a * (g - t[r])
