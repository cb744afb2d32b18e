"""fp64 model of fused sparse attention with an additive score bias (and attention dropout) -- TEST INFRASTRUCTURE.

Per stored entry e = (u, v) (duplicates count) and head h over the column window [h d, (h + 1) d):
    x_e,h = scale <Q_u,h, K_v,h> + b_e,h,  L_u,h = log sum_e exp(x_e,h),  alpha_e,h = exp(x_e,h - L_u,h),
    Z_u,h = sum_e D_e,h / (1 - p) alpha_e,h V_v,h,
with D the keep bits of tests/sparse_attention_dropout_oracle.py.  b = -inf masks an entry; a row whose entries are
all masked (or that has none) gets Z = 0, L = -inf and zero gradients.  Written per entry with index_add and
scatter_reduce, as tests/sparse_attention_oracle.py; autograd gives dQ, dK, dV and db = dLoss/dx.  fp64 on the CPU;
nothing under distributed_sddmm_b200/ imports this module.
"""
from __future__ import annotations

import numpy as np
import torch

from tests import sparse_attention_dropout_oracle as sd
from tests import sparse_attention_oracle as sa


def attention_torch(ri, ci, M, Q, K, V, B, heads, scale, p=0.0, seed=0, u0=0, v0=0):
    """(Z, L) as torch tensors: Z is M x r, L is M x heads; B is nnz x heads (entry e of head h at B[e, h]); ri + u0
    and ci + v0 are the entries' global S-rows and S-columns (the dropout mask's keys)."""
    d = Q.shape[1] // heads
    w = torch.from_numpy(sd.weights(ri.numpy() + u0, ci.numpy() + v0, heads, p, seed)) if p > 0.0 else None
    Zs, Ls = [], []
    for h in range(heads):
        win = slice(h * d, (h + 1) * d)
        x = scale * (Q[ri, win] * K[ci, win]).sum(1) + B[:, h]
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
        Zs.append(torch.zeros(M, d, dtype=x.dtype).index_add(0, ri, a[:, None] * V[ci, win]))
        Ls.append(torch.where(pos, m0 + torch.log(s1), torch.full_like(s, -torch.inf)))
    return torch.cat(Zs, 1), torch.stack(Ls, 1)


def bias_matrix(bias, nnz, heads):
    """A bias of length nnz (shared) or heads * nnz (head h at [h nnz, (h + 1) nnz)) as nnz x heads."""
    b = np.asarray(bias, np.float64)
    if len(b) == nnz:
        return np.repeat(b[:, None], heads, 1)
    assert len(b) == heads * nnz, (len(b), nnz, heads)
    return b.reshape(heads, nnz).T.copy()


def forward_np(rows, cols, M, Q, K, V, bias, heads, scale, p=0.0, seed=0, u0=0, v0=0):
    """(Z, L) as numpy; bias as bias_matrix takes it."""
    B = sa._t(bias_matrix(bias, len(rows), heads))
    with torch.no_grad():
        Z, L = attention_torch(sa._t(rows).long(), sa._t(cols).long(), M, sa._t(Q), sa._t(K), sa._t(V), B, heads, scale, p,
                               seed, u0, v0)
    return Z.numpy(), L.numpy()


def backward_np(rows, cols, M, Q, K, V, dZ, bias, heads, scale, p=0.0, seed=0, u0=0, v0=0):
    """(dQ, dK, dV, dbias) of <dZ, Z> as numpy; dbias has the bias's layout (summed over the heads for a shared
    bias)."""
    nnz = len(rows)
    q, k, v = (sa._t(x).requires_grad_() for x in (Q, K, V))
    B = sa._t(bias_matrix(bias, nnz, heads)).requires_grad_()
    Z, _ = attention_torch(sa._t(rows).long(), sa._t(cols).long(), M, q, k, v, B, heads, scale, p, seed, u0, v0)
    Z.backward(sa._t(dZ))
    g = B.grad.numpy()
    db = g.sum(1) if len(bias) == nnz else g.T.reshape(-1).copy()
    return q.grad.numpy(), k.grad.numpy(), v.grad.numpy(), db
