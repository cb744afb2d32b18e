"""fp64 model of fused sparse attention with attention dropout -- TEST INFRASTRUCTURE.

The keep bit of entry (u, v) (global S-row and S-column) in head h, restated here from include/hnh_b200.h with numpy
uint64 arithmetic (wrapping, as C's):
    key = mix64(mix64(seed + h) ^ (u << 32 | v)),  kept iff key >> 32 >= T,  T = min(ceil(p 2^32), 2^32 - 1),
with mix64 the splitmix64 finaliser.  The model is tests/sparse_attention_oracle.attention_torch on an expanded
pattern: entry e becomes its own key row, K[v_e] and D_e,h / (1 - p) V[v_e], so Z_u,h = sum_v D_uv,h / (1 - p)
alpha_uv V_v,h while L, which depends on the scores only, stays the log-sum-exp of all of them; autograd gives the
backward.  fp64 on the CPU; nothing under distributed_sddmm_b200/ imports this module.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from tests import sparse_attention_oracle as sa

_M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def mix64(z):
    """The splitmix64 finaliser on a uint64 array."""
    z = np.asarray(z, np.uint64)
    with np.errstate(over="ignore"):
        z = z + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def threshold(p):
    return min(math.ceil(p * 2.0 ** 32), 2 ** 32 - 1)


def keep(seed, h, u, v, p):
    """Keep bits (bool array) of the entries (u[i], v[i]) in head h."""
    base = mix64(np.uint64((seed + h) & 0xFFFFFFFFFFFFFFFF))
    uv = (np.asarray(u, np.uint64) << np.uint64(32)) | np.asarray(v, np.uint64)
    return (mix64(base ^ uv) >> np.uint64(32)) >= np.uint64(threshold(p))


def weights(rows, cols, heads, p, seed):
    """nnz x heads: D_uv,h / (1 - p)."""
    rows, cols = np.asarray(rows), np.asarray(cols)
    return np.stack([keep(seed, h, rows, cols, p) for h in range(heads)], 1) / (1.0 - p)


def attention_torch(ri, ci, M, Q, K, V, heads, scale, p, seed, u0=0, v0=0):
    """(Z, L) as torch tensors with dropout p and the given seed; ri + u0 and ci + v0 are the entries' global S-rows
    and S-columns."""
    d = Q.shape[1] // heads
    w = torch.from_numpy(weights(ri.numpy() + u0, ci.numpy() + v0, heads, p, seed)).repeat_interleave(d, 1)
    return sa.attention_torch(ri, torch.arange(len(ci)), M, Q, K[ci], V[ci] * w, heads, scale)


def forward_np(rows, cols, M, Q, K, V, heads, scale, p, seed, u0=0, v0=0):
    """(Z, L) as numpy for Q (M x r), K and V."""
    with torch.no_grad():
        Z, L = attention_torch(sa._t(rows).long(), sa._t(cols).long(), M, sa._t(Q), sa._t(K), sa._t(V), heads, scale, p, seed,
                               u0, v0)
    return Z.numpy(), L.numpy()


def backward_np(rows, cols, M, Q, K, V, dZ, heads, scale, p, seed, u0=0, v0=0):
    """(dQ, dK, dV) of <dZ, Z> as numpy."""
    q, k, v = (sa._t(x).requires_grad_() for x in (Q, K, V))
    Z, _ = attention_torch(sa._t(rows).long(), sa._t(cols).long(), M, q, k, v, heads, scale, p, seed, u0, v0)
    Z.backward(sa._t(dZ))
    return q.grad.numpy(), k.grad.numpy(), v.grad.numpy()
