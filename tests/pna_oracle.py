"""fp64 models of PNA (include/hnh/pna.hpp) and of multi-statistic aggregation (Distributed_Sparse::multiAggregate) --
TEST INFRASTRUCTURE.

For the stored entries (rows[i], cols[i]) of S over N nodes (duplicates count; PyG's edge_index = [cols; rows]) and a
layer of input width f, `layer_torch` is written literally from PyG's PNAConv / DegreeScalerAggregation with towers = 1,
pre_layers = post_layers = 1 and no edge features:
    h_e   = cat([x_i, x_j]) W_pre + b_pre for every entry e = (i, j)     (x_i the target row, x_j the source)
    aggregators by scatter reductions over the target (0 on a row without entries); var = mean(h^2) - mean(h)^2;
    std   = var.clamp(min=1e-5).sqrt(), masked to 0 where <= sqrt(1e-5)  (StdAggregation, semi_grad = False)
    scalers with deg = degree(rows).clamp(1); out = cat([x, scaled aggregates]) W_post + b_post, then lin
and every gradient by torch's autograd, except that min and max give each of the C entries attaining the extreme an
equal share dZ / C (the maxAggregate convention; tests/graph_sage_oracle.py says how torch's own autograd differs).
`layer_decomposed` is the form the library computes, from the statistics of z = X W_pre[f:2f] alone.  Training reuses
tests/training_oracle.py, tests/link_prediction_oracle.py and tests/graph_readout_oracle.py.  The numpy functions give
multiAggregate and its backward on their own, for the kernel and multi-rank checks.  fp64 on the CPU; nothing under
distributed_sddmm_b200/ imports this module.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from tests import link_prediction_oracle as lpo
from tests import training_oracle as tro

AGGREGATORS = ("mean", "sum", "min", "max", "var", "std")
SCALERS = ("identity", "amplification", "attenuation", "linear", "inverse_linear")
STATS = ("moments", "max", "min")
STD_EPS = 1e-5


def _t(x):
    return torch.as_tensor(np.asarray(x, np.float64))


def degree_averages(hist):
    """PyG's (avg_deg_lin, avg_deg_log) of a degree histogram, in fp64, written as PNAConv.__init__ computes them."""
    deg = torch.as_tensor(np.asarray(hist, np.float64))
    num_nodes = float(deg.sum())
    bin_degrees = torch.arange(deg.numel(), dtype=torch.float64)
    return float((bin_degrees * deg).sum()) / num_nodes, float(((bin_degrees + 1).log() * deg).sum()) / num_nodes


def _extreme(h, rows, N, mode):
    """scatter_reduce amax / amin (include_self=False; 0 on a row without entries) with the equal split of the gradient
    over the tied entries."""
    f = h.shape[1]
    index = rows[:, None].expand(len(rows), f)
    out = torch.zeros(N, f, dtype=h.dtype).scatter_reduce(0, index, h, mode, include_self=False)
    tie = (h == out[rows]).detach().to(h.dtype)
    count = torch.zeros(N, f, dtype=h.dtype).index_add(0, rows, tie)
    share = torch.zeros(N, f, dtype=h.dtype).index_add(0, rows, h * tie / count[rows].clamp(min=1))
    return out.detach() + (share - share.detach())


def _mean(h, rows, N):
    f = h.shape[1]
    return torch.zeros(N, f, dtype=h.dtype).scatter_reduce(0, rows[:, None].expand(len(rows), f), h, "mean", include_self=False)


def aggregate_torch(h, rows, N, a):
    """One of PyG's aggregations of the messages h (one row per entry) over the target rows."""
    if a == "mean":
        return _mean(h, rows, N)
    if a == "sum":
        return torch.zeros(N, h.shape[1], dtype=h.dtype).index_add(0, rows, h)
    if a in ("min", "max"):
        return _extreme(h, rows, N, "a" + a)
    var = _mean(h * h, rows, N) - _mean(h, rows, N) ** 2
    if a == "var":
        return var
    out = var.clamp(min=STD_EPS).sqrt()
    return out.masked_fill(out <= math.sqrt(STD_EPS), 0.0)


def scale_torch(out, deg, s, avg_lin, avg_log):
    """DegreeScalerAggregation's scaler s applied to out, deg already clamped to >= 1."""
    deg = deg.view(-1, 1)
    if s == "identity":
        return out
    if s == "amplification":
        return out * (torch.log(deg + 1) / avg_log)
    if s == "attenuation":
        return out * (avg_log / torch.log(deg + 1))
    if s == "linear":
        return out * (deg / avg_lin)
    return out * (avg_lin / deg)


def layer_torch(rows, cols, N, x, P, aggregators, scalers, avg_lin, avg_log):
    """One PNAConv, literally: a per-entry message cat([x_i, x_j]) W_pre + b_pre, then PyG's aggregation and scalers."""
    rows = torch.as_tensor(np.asarray(rows, np.int64))
    cols = torch.as_tensor(np.asarray(cols, np.int64))
    h = torch.cat([x[rows], x[cols]], dim=-1) @ P["pre"] + P["pre_bias"]
    out = torch.cat([aggregate_torch(h, rows, N, a) for a in aggregators], dim=-1)
    deg = torch.zeros(N, dtype=x.dtype).index_add(0, rows, torch.ones(len(rows), dtype=x.dtype)).clamp(min=1)
    out = torch.cat([scale_torch(out, deg, s, avg_lin, avg_log) for s in scalers], dim=-1)
    out = torch.cat([x, out], dim=-1) @ P["post"] + P["post_bias"]
    return out @ P["lin"] + P["lin_bias"]


def layer_decomposed(rows, cols, N, x, P, aggregators, scalers, avg_lin, avg_log):
    """The same layer as the library computes it: h_uv = c_u + z_v, every aggregate from the row statistics of z."""
    rows = torch.as_tensor(np.asarray(rows, np.int64))
    cols = torch.as_tensor(np.asarray(cols, np.int64))
    f = x.shape[1]
    c = x @ P["pre"][:f] + P["pre_bias"]
    z = x @ P["pre"][f:]
    zc = z[cols]
    d = torch.zeros(N, dtype=x.dtype).index_add(0, rows, torch.ones(len(rows), dtype=x.dtype))[:, None]
    has = d > 0
    s1 = torch.zeros(N, f, dtype=x.dtype).index_add(0, rows, zc)
    s2 = torch.zeros(N, f, dtype=x.dtype).index_add(0, rows, zc * zc)
    dd = d.clamp(min=1)
    m = s1 / dd
    var = s2 / dd - m * m
    outs = []
    for a in aggregators:
        if a == "mean":
            v = c + m
        elif a == "sum":
            v = d * c + s1
        elif a in ("min", "max"):
            v = c + _extreme(zc, rows, N, "a" + a)
        elif a == "var":
            v = var
        else:
            sd = var.clamp(min=STD_EPS).sqrt()
            v = sd.masked_fill(sd <= math.sqrt(STD_EPS), 0.0)
        outs.append(torch.where(has, v, torch.zeros_like(v)))
    out = torch.cat(outs, dim=-1)
    out = torch.cat([scale_torch(out, dd[:, 0], s, avg_lin, avg_log) for s in scalers], dim=-1)
    out = torch.cat([x, out], dim=-1) @ P["post"] + P["post_bias"]
    return out @ P["lin"] + P["lin_bias"]


def model_torch(rows, cols, N, layers, params, X, aggregators, scalers, avg_lin, avg_log, layer=layer_torch):
    """The network output; params[l] = {"pre", "pre_bias", "post", "post_bias", "lin", "lin_bias"} tensors."""
    h = X
    for l, P in enumerate(params):
        y = layer(rows, cols, N, h, P, aggregators, scalers, avg_lin, avg_log)
        h = torch.relu(y) if l + 1 < len(layers) else y
    return h


def random_params(layers, n_aggs, n_scalers, rng, scale=1.0):
    """Parameters of every layer as numpy dicts, in the library's names."""
    out = []
    for f, r in layers:
        w = (n_aggs * n_scalers + 1) * f
        out.append({"pre": rng.uniform(-1, 1, (2 * f, f)) * scale / np.sqrt(2 * f), "pre_bias": rng.uniform(-0.5, 0.5, f),
                    "post": rng.uniform(-1, 1, (w, r)) * scale / np.sqrt(w), "post_bias": rng.uniform(-0.5, 0.5, r),
                    "lin": rng.uniform(-1, 1, (r, r)) * scale / np.sqrt(r), "lin_bias": rng.uniform(-0.5, 0.5, r)})
    return out


def _leaves(params):
    return [{k: _t(v).clone().requires_grad_() for k, v in P.items()} for P in params]


def forward_backward(rows, cols, N, layers, params, X, G, *cfg):
    """(output, dL/dX, [per-layer dict of dL/d param]) for L = <output, G>, as numpy; cfg = (aggregators, scalers,
    avg_lin, avg_log)."""
    tp = _leaves(params)
    x = _t(X).clone().requires_grad_()
    out = model_torch(rows, cols, N, layers, tp, x, *cfg)
    (out * _t(G)).sum().backward()
    grads = [{k: (v.grad if v.grad is not None else torch.zeros_like(v)).numpy().copy() for k, v in P.items()} for P in tp]
    return out.detach().numpy(), x.grad.numpy().copy(), grads


def train(rows, cols, N, layers, params, X, cfg, labels, steps, **opt):
    """Node classification on the global rows; returns (per-step results, trained params as numpy dicts)."""
    tp = _leaves(params)
    x = _t(X)
    res = tro.train(lambda _: model_torch(rows, cols, N, layers, tp, x, *cfg), [v for P in tp for v in P.values()], labels, steps,
                    **opt)
    return res, [{k: v.detach().numpy().copy() for k, v in P.items()} for P in tp]


def train_link(rows, cols, N, layers, params, X, cfg, pairs, steps, **opt):
    """Link prediction over pairs = (T rows, T cols, targets); returns as train."""
    tp = _leaves(params)
    x = _t(X)
    res = lpo.link_train_step(pairs)(lambda _: model_torch(rows, cols, N, layers, tp, x, *cfg), [v for P in tp for v in P.values()],
                                     None, steps, **opt)
    return res, [{k: v.detach().numpy().copy() for k, v in P.items()} for P in tp]


# ---- multi-statistic aggregation in numpy ------------------------------------------------------------------------------
def width(which, f):
    return 2 * len(which) * f


def multi_aggregate(rows, cols, M, X, which=STATS):
    """A: the windows of `which` in the order [sum | sum of squares | max | #ties | min | #ties], 0 on an empty row."""
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    f = X.shape[1]
    Y = X[cols]
    out = []
    if "moments" in which:
        s1, s2 = np.zeros((M, f)), np.zeros((M, f))
        np.add.at(s1, rows, Y)
        np.add.at(s2, rows, Y * Y)
        out += [s1, s2]
    for name, ufunc, init in (("max", np.maximum, -np.inf), ("min", np.minimum, np.inf)):
        if name in which:
            Z = np.full((M, f), init)
            ufunc.at(Z, rows, Y)
            C = np.zeros((M, f))
            np.add.at(C, rows, (Y == Z[rows]).astype(np.float64))
            Z[C == 0] = 0.0
            out += [Z, C]
    return np.hstack(out)


def windows(A, which, f):
    """{name: window} of a state A: "s1", "s2", "max", "cmax", "min", "cmin" as present."""
    names = (["s1", "s2"] if "moments" in which else []) + (["max", "cmax"] if "max" in which else []) + \
        (["min", "cmin"] if "min" in which else [])
    return {n: A[:, i * f:(i + 1) * f] for i, n in enumerate(names)}


def multi_aggregate_backward(rows, cols, X, A, dA, N, which=STATS):
    """dX[v] = sum over the stored (u, v) of dA_s1[u] + 2 X[v] dA_s2[u] + [X[v] == max_u] dA_max[u] / C_max[u] +
    [X[v] == min_u] dA_min[u] / C_min[u] (N rows)."""
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    f = X.shape[1]
    W, dW = windows(A, which, f), windows(dA, which, f)
    Y = X[cols]
    contrib = np.zeros((len(rows), f))
    if "moments" in which:
        contrib += dW["s1"][rows] + 2.0 * Y * dW["s2"][rows]
    for name in ("max", "min"):
        if name in which:
            C = W["c" + name]
            G = np.divide(dW[name], C, out=np.zeros_like(C), where=C != 0)
            contrib += np.where(Y == W[name][rows], G[rows], 0.0)
    dX = np.zeros((N, f))
    np.add.at(dX, cols, contrib)
    return dX
