"""Autograd model of additive graph attention -- TEST INFRASTRUCTURE.

The attention of Velickovic et al. (2018) on the model of tests/gat_softmax_oracle.py: per head, with H = X W,
s = H a1 and t = H a2, the score of a stored (u, v) is x_uv = leaky_relu(s_u + t_v), alpha_u. = softmax over the
stored entries of row u of x_u., Z = S_alpha H and the head's output window = relu(Z).  fp64 on the CPU; nothing
under distributed_sddmm_b200/ imports this module.  gat_additive_forward_dense restates the forward pass with an
N x N masked torch.softmax, independently of the edge-list formulation.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from tests.gat_softmax_oracle import edge_softmax_torch, edges  # noqa: F401  (edges: re-exported for the tests)


def attention_inputs(layers, seed, scale=1.0):
    """Deterministic nonzero attention vectors: (a1[layer][head], a2[layer][head]), features_per_head long each."""
    rng = np.random.default_rng(seed + 123)
    a1 = [[scale * rng.uniform(-1, 1, fph) for _ in range(heads)] for _, fph, heads in layers]
    a2 = [[scale * rng.uniform(-1, 1, fph) for _ in range(heads)] for _, fph, heads in layers]
    return a1, a2


def gat_additive_forward_torch(ri, ci, N, layers, weights, a1, a2, alpha, X0):
    """weights[layer][head], a1 / a2[layer][head] and X0 are torch tensors; ri, ci the stored (row, col) pairs."""
    X = X0
    for (fin, fph, heads), ws, u1, u2 in zip(layers, weights, a1, a2):
        outs = []
        for h in range(heads):
            H = X @ ws[h]
            s, t = H @ u1[h], H @ u2[h]
            a = edge_softmax_torch(F.leaky_relu(s[ri] + t[ci], alpha), ri, N)
            Z = torch.zeros(N, fph, dtype=H.dtype).index_add(0, ri, a[:, None] * H[ci])
            outs.append(torch.relu(Z))
        X = torch.cat(outs, 1)
    return X


def gat_additive_forward_dense(ri, ci, N, layers, weights, a1, a2, alpha, X0):
    """The same forward pass with dense N x N scores: -inf off the pattern, torch.softmax per row (rows without
    stored entries give Z = 0)."""
    mask = torch.zeros(N, N, dtype=torch.bool)
    mask[ri, ci] = True
    has = mask.any(1)
    X = X0
    for (fin, fph, heads), ws, u1, u2 in zip(layers, weights, a1, a2):
        outs = []
        for h in range(heads):
            H = X @ ws[h]
            e = F.leaky_relu((H @ u1[h])[:, None] + (H @ u2[h])[None, :], alpha)
            e = torch.where(mask, e, torch.full_like(e, -torch.inf))
            A = torch.zeros(N, N, dtype=H.dtype)
            A[has] = torch.softmax(e[has], 1)
            outs.append(torch.relu(A @ H))
        X = torch.cat(outs, 1)
    return X


def _tensors(weights, a1, a2, grad):
    t = lambda m: torch.tensor(np.asarray(m, np.float64), requires_grad=grad)  # noqa: E731
    return ([[t(w) for w in per_layer] for per_layer in weights], [[t(v) for v in per_layer] for per_layer in a1],
            [[t(v) for v in per_layer] for per_layer in a2])


def gat_additive_backward_global(rows, cols, N, layers, weights, a1, a2, alpha, X0, grad_out):
    """Gradients of <grad_out, GAT_additive(X0)> (global matrices): (dX0, dW, da1, da2), dW / da1 / da2 indexed
    [layer][head], as numpy arrays."""
    ri, ci = edges(rows, cols, N)
    x = torch.tensor(np.asarray(X0, np.float64), requires_grad=True)
    ws, u1, u2 = _tensors(weights, a1, a2, True)
    out = gat_additive_forward_torch(ri, ci, N, layers, ws, u1, u2, alpha, x)
    out.backward(torch.from_numpy(np.asarray(grad_out, np.float64)))
    g = lambda nested: [[v.grad.numpy() for v in per_layer] for per_layer in nested]  # noqa: E731
    return x.grad.numpy(), g(ws), g(u1), g(u2)


def gat_additive_forward_global(rows, cols, N, layers, weights, a1, a2, alpha, X0):
    """The forward pass of the model above, as numpy."""
    ri, ci = edges(rows, cols, N)
    with torch.no_grad():
        ws, u1, u2 = _tensors(weights, a1, a2, False)
        X = torch.from_numpy(np.asarray(X0, np.float64))
        return gat_additive_forward_torch(ri, ci, N, layers, ws, u1, u2, alpha, X).numpy()
