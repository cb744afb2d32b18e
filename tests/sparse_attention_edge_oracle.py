"""fp64 model of fused sparse attention with edge features (and an additive score bias and attention dropout) -- TEST
INFRASTRUCTURE.

Per stored entry e = (u, v) (duplicates count) and head h over the column window [h d, (h + 1) d):
    x_e,h = scale <Q_u,h, K_v,h + E_e,h> + b_e,h,  L_u,h = log sum_e exp(x_e,h),  alpha_e,h = exp(x_e,h - L_u,h),
    Z_u,h = sum_e D_e,h / (1 - p) alpha_e,h (V_v,h + E_e,h),
with E an nnz x r matrix (row e belongs to entry e), b the bias of tests/sparse_attention_bias_oracle.py (zero when
none is given) and D the keep bits of tests/sparse_attention_dropout_oracle.py.  Written per entry as the bias model;
autograd gives dQ, dK, dV, dE and db.  fp64 on the CPU; nothing under distributed_sddmm_b200/ imports this module.
"""
from __future__ import annotations

import numpy as np
import torch

from tests import sparse_attention_bias_oracle as sb
from tests import sparse_attention_dropout_oracle as sd
from tests import sparse_attention_oracle as sa


def attention_torch(ri, ci, M, Q, K, V, E, B, heads, scale, p=0.0, seed=0, u0=0, v0=0):
    """(Z, L) as torch tensors: Z is M x r, L is M x heads; E is nnz x r, B is nnz x heads."""
    d = Q.shape[1] // heads
    w = torch.from_numpy(sd.weights(ri.numpy() + u0, ci.numpy() + v0, heads, p, seed)) if p > 0.0 else None
    Zs, Ls = [], []
    for h in range(heads):
        win = slice(h * d, (h + 1) * d)
        x = scale * (Q[ri, win] * (K[ci, win] + E[:, win])).sum(1) + B[:, h]
        m = torch.full((M,), -torch.inf, dtype=x.dtype).scatter_reduce(0, ri, x.detach(), "amax", include_self=True)
        has = torch.isfinite(m)
        m0 = torch.where(has, m, torch.zeros_like(m))
        ex = torch.exp(x - m0[ri])
        s = torch.zeros(M, dtype=x.dtype).index_add(0, ri, ex)
        pos = s > 0
        s1 = torch.where(pos, s, torch.ones_like(s))
        a = ex / s1[ri]
        if w is not None:
            a = a * w[:, h]
        Zs.append(torch.zeros(M, d, dtype=x.dtype).index_add(0, ri, a[:, None] * (V[ci, win] + E[:, win])))
        Ls.append(torch.where(pos, m0 + torch.log(s1), torch.full_like(s, -torch.inf)))
    return torch.cat(Zs, 1), torch.stack(Ls, 1)


def _bias(bias, nnz, heads):
    return sa._t(np.zeros((nnz, heads)) if bias is None else sb.bias_matrix(bias, nnz, heads))


def forward_np(rows, cols, M, Q, K, V, E, heads, scale, p=0.0, seed=0, u0=0, v0=0, bias=None):
    """(Z, L) as numpy; bias None or as bias_matrix takes it."""
    with torch.no_grad():
        Z, L = attention_torch(sa._t(rows).long(), sa._t(cols).long(), M, sa._t(Q), sa._t(K), sa._t(V), sa._t(E),
                               _bias(bias, len(rows), heads), heads, scale, p, seed, u0, v0)
    return Z.numpy(), L.numpy()


def backward_np(rows, cols, M, Q, K, V, E, dZ, heads, scale, p=0.0, seed=0, u0=0, v0=0, bias=None):
    """(dQ, dK, dV, dE, dbias) of <dZ, Z> as numpy; dbias has the bias's layout (None without a bias)."""
    nnz = len(rows)
    q, k, v, e = (sa._t(x).requires_grad_() for x in (Q, K, V, E))
    B = _bias(bias, nnz, heads).requires_grad_()
    Z, _ = attention_torch(sa._t(rows).long(), sa._t(cols).long(), M, q, k, v, e, B, heads, scale, p, seed, u0, v0)
    Z.backward(sa._t(dZ))
    db = None
    if bias is not None:
        g = B.grad.numpy()
        db = g.sum(1) if len(bias) == nnz else g.T.reshape(-1).copy()
    return q.grad.numpy(), k.grad.numpy(), v.grad.numpy(), e.grad.numpy(), db
