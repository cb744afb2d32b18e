"""Autograd model of GATv2 attention -- TEST INFRASTRUCTURE.

GATv2 with shared weights (Brody, Alon and Yahav 2022) on the model of tests/gat_softmax_oracle.py: per head, with
H = X W and a the head's attention vector, the score of a stored (u, v) is x_uv = sum_k a_k leaky_relu(H_uk + H_vk),
alpha_u. = softmax over the stored entries of row u of x_u., Z = S_alpha H and the head's output window = relu(Z).
fp64 on the CPU; nothing under distributed_sddmm_b200/ imports this module.  gatv2_forward_dense restates the forward
pass with an N x N masked torch.softmax, independently of the edge-list formulation.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from tests.gat_softmax_oracle import edge_softmax_torch, edges  # noqa: F401  (edges: re-exported for the tests)


def attention_inputs(layers, seed, scale=1.0):
    """Deterministic nonzero attention vectors a[layer][head], features_per_head long each."""
    rng = np.random.default_rng(seed + 321)
    return [[scale * rng.uniform(-1, 1, fph) for _ in range(heads)] for _, fph, heads in layers]


def gatv2_forward_torch(ri, ci, N, layers, weights, a, alpha, X0):
    """weights[layer][head], a[layer][head] and X0 are torch tensors; ri, ci the stored (row, col) pairs."""
    X = X0
    for (fin, fph, heads), ws, av in zip(layers, weights, a):
        outs = []
        for h in range(heads):
            H = X @ ws[h]
            x = F.leaky_relu(H[ri] + H[ci], alpha) @ av[h]
            att = edge_softmax_torch(x, ri, N)
            Z = torch.zeros(N, fph, dtype=H.dtype).index_add(0, ri, att[:, None] * H[ci])
            outs.append(torch.relu(Z))
        X = torch.cat(outs, 1)
    return X


def gatv2_forward_dense(ri, ci, N, layers, weights, a, alpha, X0):
    """The same forward pass with dense N x N scores: -inf off the pattern, torch.softmax per row (rows without
    stored entries give Z = 0)."""
    mask = torch.zeros(N, N, dtype=torch.bool)
    mask[ri, ci] = True
    has = mask.any(1)
    X = X0
    for (fin, fph, heads), ws, av in zip(layers, weights, a):
        outs = []
        for h in range(heads):
            H = X @ ws[h]
            e = F.leaky_relu(H[:, None, :] + H[None, :, :], alpha) @ av[h]
            e = torch.where(mask, e, torch.full_like(e, -torch.inf))
            A = torch.zeros(N, N, dtype=H.dtype)
            A[has] = torch.softmax(e[has], 1)
            outs.append(torch.relu(A @ H))
        X = torch.cat(outs, 1)
    return X


def _tensors(weights, a, grad):
    t = lambda m: torch.tensor(np.asarray(m, np.float64), requires_grad=grad)  # noqa: E731
    return [[t(w) for w in per_layer] for per_layer in weights], [[t(v) for v in per_layer] for per_layer in a]


def gatv2_backward_global(rows, cols, N, layers, weights, a, alpha, X0, grad_out):
    """Gradients of <grad_out, GATv2(X0)> (global matrices): (dX0, dW, da), dW / da indexed [layer][head], as numpy."""
    ri, ci = edges(rows, cols, N)
    x = torch.tensor(np.asarray(X0, np.float64), requires_grad=True)
    ws, av = _tensors(weights, a, True)
    out = gatv2_forward_torch(ri, ci, N, layers, ws, av, alpha, x)
    out.backward(torch.from_numpy(np.asarray(grad_out, np.float64)))
    g = lambda nested: [[v.grad.numpy() for v in per_layer] for per_layer in nested]  # noqa: E731
    return x.grad.numpy(), g(ws), g(av)


def gatv2_forward_global(rows, cols, N, layers, weights, a, alpha, X0):
    """The forward pass of the model above, as numpy."""
    ri, ci = edges(rows, cols, N)
    with torch.no_grad():
        ws, av = _tensors(weights, a, False)
        X = torch.from_numpy(np.asarray(X0, np.float64))
        return gatv2_forward_torch(ri, ci, N, layers, ws, av, alpha, X).numpy()


def scores_np(R, Y, rows, cols, a, alpha):
    """x_i = sum_k a_k leaky_relu(R[rows_i, k] + Y[cols_i, k]) for edge lists, as numpy (the kernel-level reference)."""
    z = R[rows] + Y[cols]
    return np.where(z > 0, z, alpha * z) @ a


def grad_np(R, Y, rows, cols, g, a, alpha):
    """(dR, da) of the kernel-level backward: dR[u] = a o sum over entries of row u of g sigma'(z), da = sum g sigma(z)."""
    z = R[rows] + Y[cols]
    dR = np.zeros_like(R)
    np.add.at(dR, rows, g[:, None] * np.where(z > 0, 1.0, alpha))
    return dR * a, (g[:, None] * np.where(z > 0, z, alpha * z)).sum(0)
