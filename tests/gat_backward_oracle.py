"""Autograd model of the GAT backward pass -- TEST INFRASTRUCTURE.

The global model of oracle.hnh_oracle.gat_forward_global (the forward pass pinned to the reference's gat.hpp),
restated in torch on the CPU in fp64 and differentiated with torch.autograd.  torch.relu and F.leaky_relu give the
derivative conventions at 0 that the library uses (relu'(0) = 0, leaky_relu'(0) = alpha).  Nothing under
distributed_sddmm_b200/ imports this module.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F


def edges(rows, cols, N):
    """The stored (row, col) pairs of the N x N pattern, unique, sorted by (row, col), as int64 tensors."""
    key = np.unique(np.asarray(rows, np.int64) * N + np.asarray(cols, np.int64))
    return torch.from_numpy(key // N), torch.from_numpy(key % N)


def gat_forward_torch(ri, ci, N, layers, weights, alpha, X0):
    """Per head: H = X W; e_uv = <H_u, H_v> on every stored (u, v); a = leaky_relu(e); Z = S_a H; the head's
    output window = relu(Z).  weights[layer][head] and X0 are torch tensors."""
    X = X0
    for (fin, fph, heads), ws in zip(layers, weights):
        outs = []
        for h in range(heads):
            H = X @ ws[h]
            e = (H[ri] * H[ci]).sum(1)
            a = F.leaky_relu(e, alpha)
            Z = torch.zeros(N, fph, dtype=H.dtype).index_add(0, ri, a[:, None] * H[ci])
            outs.append(torch.relu(Z))
        X = torch.cat(outs, 1)
    return X


def gat_backward_global(rows, cols, N, layers, weights, alpha, X0, grad_out):
    """Gradients of <grad_out, GAT(X0)> (global matrices): returns (dX0, dW[layer][head]) as numpy arrays."""
    ri, ci = edges(rows, cols, N)
    x = torch.tensor(np.asarray(X0, np.float64), requires_grad=True)
    ws = [[torch.tensor(np.asarray(w, np.float64), requires_grad=True) for w in per_layer] for per_layer in weights]
    out = gat_forward_torch(ri, ci, N, layers, ws, alpha, x)
    out.backward(torch.from_numpy(np.asarray(grad_out, np.float64)))
    return x.grad.numpy(), [[w.grad.numpy() for w in per_layer] for per_layer in ws]


def gat_forward_global_torch(rows, cols, N, layers, weights, alpha, X0):
    """The forward pass of the model above, as numpy."""
    ri, ci = edges(rows, cols, N)
    with torch.no_grad():
        ws = [[torch.from_numpy(np.asarray(w, np.float64)) for w in per_layer] for per_layer in weights]
        return gat_forward_torch(ri, ci, N, layers, ws, alpha, torch.from_numpy(np.asarray(X0, np.float64))).numpy()
