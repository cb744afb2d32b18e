"""fp64 model of the graph transformer written per stored entry -- TEST INFRASTRUCTURE.

The network of tests/graph_transformer_oracle.py (ffn = 0) and tests/graph_transformer_block_oracle.py (ffn > 0),
restated over the stored entries instead of a dense N x N (x d) score matrix, so that it runs on graphs of thousands of
nodes with rows of thousands of entries.  Per layer with input X, H heads of width d and r = H d:
    Q, K, V, R = X W_q + b_q, X W_k + b_k, X W_v + b_v, X W_s + b_s,   E = attr W_e  (nnz x r; zero without edge features)
    M = the Z of tests/sparse_attention_edge_oracle.attention_torch(Q, K, V, E, bias 0, scale 1 / sqrt(d), p, seed_l)
    Y = M + R, or with the gate  beta_u = sigmoid(w_beta . [M_u, R_u, M_u - R_u]),  Y = beta R + (1 - beta) M
    X_next = gbo.block(Y) with ffn > 0, else ReLU(Y) except after the last layer
with seed_l = seed + the heads of the earlier layers.  Every stored copy of a duplicated pair is its own entry, which
is the dense models' log count term; rows without entries have M = 0, so Y = R (beta R with the gate).  attr is per
stored entry (nnz x e), in the order of rows and cols.  fp64 on the CPU; nothing under distributed_sddmm_b200/ imports
this module.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from tests import graph_transformer_block_oracle as gbo
from tests import graph_transformer_oracle as gto
from tests import link_prediction_oracle as lpo
from tests import sparse_attention_edge_oracle as se
from tests import training_oracle as tro


def layer_torch(ri, ci, N, layer, P, X, attr, beta, p, seed):
    """The layer's Y (before the ReLU or the block) as a torch tensor."""
    _, d, H = layer
    Q, K, V, R = (X @ P[n] + P[n + "_bias"] for n in gto.PROJECTIONS)
    E = attr @ P["edge"] if attr is not None else torch.zeros(len(ri), H * d, dtype=X.dtype)
    M, _ = se.attention_torch(ri, ci, N, Q, K, V, E, torch.zeros(len(ri), H, dtype=X.dtype), H, 1 / math.sqrt(d), p, seed)
    if beta:
        b = torch.sigmoid(torch.cat([M, R, M - R], 1) @ P["beta"])[:, None]
        return b * R + (1 - b) * M
    return M + R


def model_torch(rows, cols, N, layers, params, X, attr=None, beta=False, p=0.0, seed=0, ffn=0, eps=1e-5):
    """Output of the network (N x r_last) as a torch tensor.  params: per layer a dict name -> tensor; attr: an nnz x e
    tensor or None; ffn > 0: transformer blocks (their width comes from the parameters)."""
    ri, ci = torch.as_tensor(np.asarray(rows, np.int64)), torch.as_tensor(np.asarray(cols, np.int64))
    s = seed
    for l, layer in enumerate(layers):
        Y = layer_torch(ri, ci, N, layer, params[l], X, attr, beta, p, s)
        X = gbo.block(Y, params[l], eps) if ffn else torch.relu(Y) if l + 1 < len(layers) else Y
        s += layer[2]
    return X


def _attr(attr):
    return gto._t(attr) if attr is not None else None


def forward_np(rows, cols, N, layers, params, X, attr=None, beta=False, p=0.0, seed=0, ffn=0, eps=1e-5):
    """The network output as numpy; attr: per-entry attributes (nnz x e) or None."""
    with torch.no_grad():
        return model_torch(rows, cols, N, layers, [{k: gto._t(v) for k, v in P.items()} for P in params], gto._t(X),
                           _attr(attr), beta, p, seed, ffn, eps).numpy()


def backward_np(rows, cols, N, layers, params, X, G, attr=None, beta=False, p=0.0, seed=0, ffn=0, eps=1e-5):
    """(output, dX, [per layer dict name -> gradient]) of <G, output> as numpy."""
    tp = [{k: gto._t(v).requires_grad_() for k, v in P.items()} for P in params]
    x = gto._t(X).requires_grad_()
    out = model_torch(rows, cols, N, layers, tp, x, _attr(attr), beta, p, seed, ffn, eps)
    out.backward(gto._t(G))
    return out.detach().numpy(), x.grad.numpy(), [{k: v.grad.numpy() for k, v in P.items()} for P in tp]


def _train(step, rows, cols, N, layers, params, X, targets, steps, attr, beta, ffn, dropout, seeds, eps, opt):
    tp = tro._leaves(params)
    A, x = _attr(attr), gto._t(X)
    seeds = seeds or [0] * steps

    def forward(t):
        return model_torch(rows, cols, N, layers, tp, x, A, beta, dropout, seeds[t], ffn, eps)

    res = step(forward, [v for P in tp for v in P.values()], targets, steps, **opt)
    return res, [{k: v.detach().numpy().copy() for k, v in P.items()} for P in tp]


def train_gt(rows, cols, N, layers, params, X, labels, steps, attr=None, beta=False, ffn=0, dropout=0.0, seeds=None, eps=1e-5,
             **opt):
    """tests/training_oracle.train_gt on this model: (per-step results, trained params as numpy dicts); seeds[t] is the
    dropout seed of step t."""
    return _train(tro.train, rows, cols, N, layers, params, X, labels, steps, attr, beta, ffn, dropout, seeds, eps, opt)


def link_train_gt(rows, cols, N, layers, params, X, pairs, steps, attr=None, beta=False, ffn=0, dropout=0.0, seeds=None,
                  eps=1e-5, **opt):
    """tests/link_prediction_oracle.train_gt on this model: the link loss over pairs = (T rows, T cols, targets)."""
    return _train(lpo.link_train_step(pairs), rows, cols, N, layers, params, X, None, steps, attr, beta, ffn, dropout, seeds,
                  eps, opt)
