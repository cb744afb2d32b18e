"""The PNA, GIN and GINE cases of the skewed-graph tests (mp_skewed_worker.GNN_CONFIGS and the gine_int op case),
checked without a GPU: that they reach the kernels they are aimed at, and that no pass can be decided by a
floating-point tie or threshold.

  * PNA's literal per-edge model (pna_oracle.layer_torch, ties of min and max on h = c_u + z_v) equals the decomposed
    form the library computes (layer_decomposed, ties on z) to 1e-12 in the output, dX and every parameter gradient.
  * No std cell of any PNA layer has var within 1e-9 relative of PyG's clamp of 1e-5, so the clamp and the mask
    decide no cell by rounding.
  * Every configuration aggregates at the widths it names, by HNH_DISPATCH_R and kWindow as the CUDA sources state them.
  * gine_int: X_v + E_i == 0 on the hub row, and integer sums far below 2^53 (exact on any order)."""
import os
import re

import numpy as np
import pytest
import torch

from tests import gin_oracle as go
from tests import mp_skewed_worker as W
from tests import pna_oracle as po
from tests.skewed_graph import DEFAULT_N, landmarks, skewed_tuples
from tests.test_skewed_graphs_multirank_gpu import SEED

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "distributed_sddmm_b200", "csrc")
PNA_CONFIGS = sorted(k for k, v in W.GNN_CONFIGS.items() if v["model"] == "pna")


def _src(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def aggregation_tables():
    """The widths of HNH_DISPATCH_R (row_gather.cuh) and the column window of pna.cu and gine.cu."""
    row = re.search(r"#define HNH_DISPATCH_R\(r, CALL, FALLBACK\)(.*?)default:", _src("row_gather.cuh"), re.S)
    assert row, "HNH_DISPATCH_R"
    windows = [re.search(r"constexpr int kWindow = (\d+);", _src(f)) for f in ("pna.cu", "gine.cu")]
    assert all(windows), "kWindow"
    assert windows[0].group(1) == windows[1].group(1)
    return sorted(int(w) for w in re.findall(r"case (\d+):", row.group(1))), int(windows[0].group(1))


def path(width, table, window):
    """The aggregation path of a width: one table window, several column windows, or the generic kernels."""
    if width > window:
        return "windows"
    return "table" if width in table else "generic"


_GRAPH = {}


def graph():
    if not _GRAPH:
        r, c = (x.astype(np.int64) for x in skewed_tuples(DEFAULT_N, DEFAULT_N, SEED))
        order = np.lexsort((c, r))
        _GRAPH["g"] = (DEFAULT_N, r[order], c[order])
    return _GRAPH["g"]


@pytest.mark.parametrize("name", sorted(W.GNN_CONFIGS))
def test_configurations_reach_their_aggregation_paths(name):
    table, window = aggregation_tables()
    cfg = W.GNN_CONFIGS[name]
    widths = [l[0] for l in cfg["layers"]]  # every model aggregates its layer input (PNA: z = X W_pre[f:2f], f wide)
    got = tuple(path(w, table, window) for w in widths)
    assert got == tuple(cfg["reach"]), (name, "aggregates at", widths, "reaching", got, "not", cfg["reach"], table, window)
    layers = cfg["layers"]
    assert all(layers[l + 1][0] == layers[l][-1] for l in range(len(layers) - 1)), name
    if name.endswith("_table"):  # every 128-bit width of 64 and above, in order
        assert widths == [w for w in table if w >= 64], (name, widths, table)
    if name == "pna_wide":  # a full window and a remainder
        assert widths[0] > window and widths[0] % window
    if name.endswith("_odd"):
        assert all(w % 2 for w in widths), name
    if name == "pna_all":
        assert tuple(cfg["aggregators"]) == po.AGGREGATORS and tuple(cfg["scalers"]) == po.SCALERS
    if cfg["model"] == "gin":
        assert cfg["edge_dim"] == (0 if name.startswith("gin_") else 3 if name == "gine_table" else 2), name
    assert path(W.GINE_INT_WIDTH, table, window) == "table"


def _pna(name):
    N, rows, cols = graph()
    cfg = W.gnn_config(dict(gnn=name))
    params, X, G = W.gnn_inputs(N, cfg, SEED)
    hist = np.bincount(np.bincount(rows, minlength=N))
    return N, rows, cols, cfg, params, X, G, (cfg["aggregators"], cfg["scalers"], *po.degree_averages(hist))


@pytest.mark.parametrize("name", PNA_CONFIGS)
def test_pna_per_edge_model_equals_the_decomposed_one(name):
    """Output, dX and every parameter gradient to 1e-12 of their largest entry: min and max tie on z exactly where they
    tie on h, and the moments of h and of z give the same aggregates."""
    N, rows, cols, cfg, params, X, G, oracle = _pna(name)
    results = []
    for layer in (po.layer_torch, po.layer_decomposed):
        tp = po._leaves(params)
        x = po._t(X).clone().requires_grad_()
        out = po.model_torch(rows, cols, N, cfg["layers"], tp, x, *oracle, layer=layer)
        (out * po._t(G)).sum().backward()
        results.append([out.detach().numpy(), x.grad.numpy()] + [v.grad.numpy() for P in tp for v in P.values()])
    for i, (a, b) in enumerate(zip(*results)):
        assert np.abs(b).max() > 0, (name, i)
        assert np.abs(a - b).max() <= 1e-12 * np.abs(b).max(), (name, i, np.abs(a - b).max() / np.abs(b).max())


@pytest.mark.parametrize("name", [n for n in PNA_CONFIGS if "std" in W.GNN_CONFIGS[n]["aggregators"]])
def test_no_std_cell_sits_at_the_clamp(name):
    """var = S2 / d - (S1 / d)^2 of z on every row with entries, in every layer (the layer inputs from the model's own
    forward): never within 1e-9 relative of 1e-5."""
    N, rows, cols, cfg, params, X, G, oracle = _pna(name)
    deg = np.bincount(rows, minlength=N).astype(np.float64)
    has = deg > 0
    h = po._t(X)
    near = 0
    with torch.no_grad():
        for l, P in enumerate(params):
            f = cfg["layers"][l][0]
            z = h.numpy() @ P["pre"][f:]
            s1, s2 = np.zeros((N, f)), np.zeros((N, f))
            np.add.at(s1, rows, z[cols])
            np.add.at(s2, rows, z[cols] ** 2)
            m = s1[has] / deg[has, None]
            var = s2[has] / deg[has, None] - m * m
            near += int((np.abs(var - po.STD_EPS) <= 1e-9 * po.STD_EPS).sum())
            assert (var > po.STD_EPS).any() and (var < po.STD_EPS).any(), (name, l)  # both sides of the clamp are met
            y = po.layer_torch(rows, cols, N, h, {k: po._t(v) for k, v in P.items()}, *oracle)
            h = torch.relu(y) if l + 1 < len(params) else y
    assert near == 0, (name, near)


def test_pna_hub_rows_reach_the_scalers_at_their_full_degree():
    """The degree the scalers read is a whole row's over every column block: above 2800 on both wide hubs, each of
    them with more than 500 entries in every one of the 4 column blocks."""
    N, rows, cols = graph()
    lm = landmarks(N, N)
    for u in lm["wide_hubs"]:
        mine = cols[rows == u]
        assert len(mine) > 2800 and all((mine // lm["w"] == b).sum() > 500 for b in range(4)), u


def test_gine_int_inputs_meet_the_strict_mask_and_stay_exact():
    N, rows, cols = graph()
    f = W.GINE_INT_WIDTH
    X, dA = W.gine_int_inputs(N, f, SEED)
    E = go.edge_rows(rows, cols, f)
    assert np.array_equal(X, np.round(X)) and np.array_equal(E, np.round(E)) and np.array_equal(dA, np.round(dA))
    hub = rows == landmarks(N, N)["wide_hubs"][0]
    zero = X[cols] + E == 0
    assert zero[hub].sum() > 100 and (X[cols] + E > 0)[hub].any() and (X[cols] + E < 0)[hub].any()
    A = go.edge_relu_aggregate(rows, cols, N, X, E)
    dX, dE = go.edge_relu_aggregate_backward(rows, cols, X, E, dA, N)
    # the largest partial sum of any order is below the sum of absolute values, far below 2^53
    bound_A = np.zeros((N, f))
    np.add.at(bound_A, rows, np.abs(X[cols] + E))
    bound_dX = np.zeros((N, f))
    np.add.at(bound_dX, cols, np.abs(dA[rows]))
    assert bound_A.max() < 2 ** 30 and bound_dX.max() < 2 ** 30
    assert np.abs(A).max() > 0 and np.abs(dX).max() > 0 and not dE[zero].any()


def test_readout_batch_holds_what_the_graph_cases_need():
    """Graph 0 spans all 4 row blocks with a hub row; graph 1 is two rows without entries and with equal inputs, in the
    first and the last row block (and in different blocks of 2); graph 2 is empty."""
    N, rows, _ = graph()
    batch, G, labels = W.readout_batch(N, SEED)
    q = -(-N // 4)
    g0 = np.flatnonzero(batch == 0)
    assert len(np.unique(g0 // q)) == 4 and landmarks(N, N)["wide_hubs"][0] in g0
    assert not (batch == 2).any() and len(labels) == G and (labels < 0).sum() == 2
    t = list(W.TIE_ROWS)
    assert np.array_equal(np.flatnonzero(batch == 1), t) and not np.bincount(rows, minlength=N)[t].any()
    assert t[0] // q != t[1] // q and t[0] // (2 * q) != t[1] // (2 * q)
    for name in ("pna_table", "gin_table"):
        _, X, _ = W.gnn_inputs(N, W.gnn_config(dict(gnn=name)), SEED)
        assert np.array_equal(X[t[0]], X[t[1]])
