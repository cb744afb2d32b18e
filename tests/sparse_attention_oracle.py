"""fp64 model of fused sparse attention -- TEST INFRASTRUCTURE.

Per entry (u, v) of S's pattern (duplicates count, S's values are not read) and head h over the column window
[h d, (h + 1) d):  x_uv = scale <Q_u,h, K_v,h>, L_u,h = log sum_v exp(x_uv) (-inf for a row without entries),
alpha_uv = exp(x_uv - L_u,h), Z_u,h = sum_v alpha_uv V_v,h (0 for a row without entries).  Written per entry with
index_add and scatter_reduce, as tests/gat_softmax_oracle.py; autograd gives the backward.  fp64 on the CPU; nothing
under distributed_sddmm_b200/ imports this module.
"""
from __future__ import annotations

import numpy as np
import torch


def attention_torch(ri, ci, M, Q, K, V, heads, scale):
    """(Z, L) as torch tensors: Z is M x r, L is M x heads."""
    d = Q.shape[1] // heads
    Zs, Ls = [], []
    for h in range(heads):
        w = slice(h * d, (h + 1) * d)
        x = scale * (Q[ri, w] * K[ci, w]).sum(1)
        m = torch.full((M,), -torch.inf, dtype=x.dtype).scatter_reduce(0, ri, x.detach(), "amax", include_self=True)
        has = torch.isfinite(m)
        m0 = torch.where(has, m, torch.zeros_like(m))
        ex = torch.exp(x - m0[ri])
        s = torch.zeros(M, dtype=x.dtype).index_add(0, ri, ex)
        a = ex / s[ri]
        Zs.append(torch.zeros(M, d, dtype=x.dtype).index_add(0, ri, a[:, None] * V[ci, w]))
        s1 = torch.where(has, s, torch.ones_like(s))
        Ls.append(torch.where(has, m0 + torch.log(s1), torch.full_like(s, -torch.inf)))
    return torch.cat(Zs, 1), torch.stack(Ls, 1)


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x, np.float64))


def forward_np(rows, cols, M, Q, K, V, heads, scale):
    """(Z, L) as numpy for global Q (M x r), K and V (N x r)."""
    with torch.no_grad():
        Z, L = attention_torch(_t(rows).long(), _t(cols).long(), M, _t(Q), _t(K), _t(V), heads, scale)
    return Z.numpy(), L.numpy()


def backward_np(rows, cols, M, Q, K, V, dZ, heads, scale):
    """(dQ, dK, dV) of <dZ, Z> as numpy."""
    q, k, v = (_t(x).requires_grad_() for x in (Q, K, V))
    Z, _ = attention_torch(_t(rows).long(), _t(cols).long(), M, q, k, v, heads, scale)
    Z.backward(_t(dZ))
    return q.grad.numpy(), k.grad.numpy(), v.grad.numpy()


def dense_masked_np(rows, cols, M, N, Q, K, V, heads, scale):
    """Z by a dense masked torch.softmax(...) @ V per head, on rows with entries (zeros elsewhere); duplicate pairs
    count once per copy (their multiplicity adds log(count) to the score)."""
    d = Q.shape[1] // heads
    count = np.zeros((M, N))
    np.add.at(count, (rows, cols), 1.0)
    cnt = torch.from_numpy(count)
    Z = torch.zeros(M, Q.shape[1], dtype=torch.float64)
    has = cnt.sum(1) > 0
    for h in range(heads):
        w = slice(h * d, (h + 1) * d)
        x = scale * _t(Q)[:, w] @ _t(K)[:, w].T + torch.log(cnt)
        x = torch.where(cnt > 0, x, torch.full_like(x, -torch.inf))
        Z[has, w] = torch.softmax(x[has], 1) @ _t(V)[:, w]
    return Z.numpy()
