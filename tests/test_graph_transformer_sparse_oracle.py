"""The per-entry fp64 model of the graph transformer (tests/graph_transformer_sparse_oracle.py) against the dense
models it restates (tests/graph_transformer_oracle.py, tests/graph_transformer_block_oracle.py), forward, backward and
in training; and the skewed-graph configurations of tests/mp_skewed_worker.GT_CONFIGS against the kernels' tables,
read from the CUDA sources, so that a changed table names the configuration that no longer reaches its path.  No GPU."""
import os
import re

import numpy as np
import pytest

from tests import graph_transformer_block_oracle as gbo
from tests import graph_transformer_oracle as gto
from tests import graph_transformer_sparse_oracle as gts
from tests import link_prediction_oracle as lpo
from tests import training_oracle as tro
from tests.mp_graph_transformer_worker import attr_of
from tests.mp_skewed_worker import GT_CONFIGS
from tests.skewed_graph import DEFAULT_N, HUB_MIN, landmarks, skewed_tuples

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "distributed_sddmm_b200", "csrc")


def graph(seed, N=40):
    """A small pattern with empty rows, duplicates (one pair stored three times) and a row of many entries."""
    rng = np.random.default_rng(seed)
    rows, cols = rng.integers(0, N, 4 * N), rng.integers(0, N, 4 * N)
    keep = rows % 7 != 3  # rows without entries
    rows, cols = rows[keep], cols[keep]
    rows = np.concatenate([rows, [5, 5, 5], np.full(N // 2, 2)])
    cols = np.concatenate([cols, [9, 9, 9], np.arange(0, N, 2)])
    assert (np.bincount(rows, minlength=N) == 0).any()
    return rows.astype(np.int64), cols.astype(np.int64), N


def err(got, want):
    return np.abs(got - want).max() / max(np.abs(want).max(), 1e-300)


CONFIGS = [
    # layers, edge_dim, beta, ffn, dropout
    ([(6, 4, 2)], 0, False, 0, 0.0),
    ([(6, 4, 2), (8, 3, 3)], 3, True, 0, 0.3),
    ([(6, 4, 2), (8, 3, 3), (9, 8, 1)], 2, False, 0, 0.3),
    ([(6, 4, 2)], 3, True, 1, 0.3),
    ([(5, 3, 2), (6, 4, 2)], 0, True, 2, 0.0),
    ([(6, 4, 2), (8, 3, 3), (9, 5, 1)], 2, True, 1, 0.3),
]


@pytest.mark.parametrize("i", range(len(CONFIGS)))
def test_matches_the_dense_models(i):
    layers, edge_dim, beta, ffn, p = CONFIGS[i]
    rows, cols, N = graph(i)
    rng = np.random.default_rng(100 + i)
    params = gbo.random_params(layers, edge_dim, beta, ffn, rng)
    X = rng.uniform(-1, 1, (N, layers[0][0]))
    G = rng.uniform(-1, 1, (N, layers[-1][1] * layers[-1][2]))
    attr = attr_of(rows, cols, edge_dim) if edge_dim else None
    dense = gbo if ffn else gto
    kw = dict(attr=attr, beta=beta, p=p, seed=7)
    want = dense.forward_np(rows, cols, N, layers, params, X, **kw)
    want_dX, want_dP = dense.backward_np(rows, cols, N, layers, params, X, G, **kw)
    got = gts.forward_np(rows, cols, N, layers, params, X, ffn=ffn, **kw)
    out, dX, dP = gts.backward_np(rows, cols, N, layers, params, X, G, ffn=ffn, **kw)
    assert np.abs(want).max() > 0 and err(got, want) < 1e-13 and np.array_equal(out, got)
    assert err(dX, want_dX) < 1e-13
    for l, grads in enumerate(want_dP):
        assert set(dP[l]) == set(grads)
        scale = max(np.abs(g).max() for g in grads.values())
        for k, g in grads.items():  # key_bias: 0 up to rounding, measured against the layer's largest gradient
            assert np.abs(dP[l][k] - g).max() <= 1e-13 * max(np.abs(g).max(), scale), (i, l, k)
    if p:  # dropout is in both, drawn at seed + the heads of the earlier layers
        assert err(gts.forward_np(rows, cols, N, layers, params, X, ffn=ffn, **dict(kw, p=0.0)), want) > 1e-6


def test_rows_without_entries_take_the_skip():
    rows, cols, N = graph(3)
    layers = [(6, 4, 2)]
    rng = np.random.default_rng(5)
    for beta in (False, True):
        params = gbo.random_params(layers, 3, beta, 0, rng)
        X = rng.uniform(-1, 1, (N, 6))
        Y = gts.forward_np(rows, cols, N, layers, params, X, attr=attr_of(rows, cols, 3), beta=beta, p=0.3, seed=1)
        P = params[0]
        R = X @ P["skip"] + P["skip_bias"]
        empty = np.bincount(rows, minlength=N) == 0
        if beta:  # M = 0: beta = sigmoid(w2 . R - w3 . R)
            r = R.shape[1]
            b = 1 / (1 + np.exp(-(R @ P["beta"][r:2 * r] - R @ P["beta"][2 * r:])))
            R = b[:, None] * R
        assert np.abs(Y[empty] - R[empty]).max() < 1e-14


STEP_CASES = [([(6, 4, 2), (8, 5, 1)], 3, True, 1, 0.3, 0.05), ([(6, 4, 2), (8, 3, 2)], 0, False, 0, 0.0, None)]


@pytest.mark.parametrize("i", range(len(STEP_CASES)))
def test_train_steps_match_the_dense_models(i):
    layers, edge_dim, beta, ffn, p, clip = STEP_CASES[i]
    rows, cols, N = graph(20 + i)
    rng = np.random.default_rng(200 + i)
    params = gbo.random_params(layers, edge_dim, beta, ffn, rng)
    X = rng.uniform(-1, 1, (N, layers[0][0]))
    C = layers[-1][1] * layers[-1][2]
    labels = rng.integers(0, C, N)
    labels[rng.random(N) < 0.3] = -1
    kw = dict(attr=attr_of(rows, cols, edge_dim) if edge_dim else None, beta=beta, ffn=ffn, dropout=p, seeds=[3, 10, 17],
              lr=1e-2, lrs=[1e-2, 3e-2, 2e-2], weight_decay=0.01, max_grad_norm=clip)
    tr, tc = rng.integers(0, N, 90), rng.integers(0, N, 90)
    y = rng.choice([0.0, 1.0, 0.25], 90)
    for (got, gp), (want, wp) in ((gts.train_gt(rows, cols, N, layers, params, X, labels, 3, **kw),
                                   tro.train_gt(rows, cols, N, layers, params, X, labels, 3, **kw)),
                                  (gts.link_train_gt(rows, cols, N, layers, params, X, (tr, tc, y), 3, **kw),
                                   lpo.train_gt(rows, cols, N, layers, params, X, (tr, tc, y), 3, **kw))):
        for g, w in zip(got, want):
            assert abs(g[0] - w[0]) <= 1e-13 * abs(w[0]) and g[1:3] == w[1:3] and abs(g[3] - w[3]) <= 1e-12 * w[3], (g, w)
        if clip:
            assert any(w[3] > clip for w in want)
        for l, P in enumerate(wp):
            for k, w in P.items():
                assert np.abs(gp[l][k] - w).max() <= 1e-11 * max(np.abs(w).max(), 1.0), (i, l, k)


# ---- what the skewed-graph configurations reach ----------------------------------------------------------------------
def _src(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def kernel_tables():
    """The constants the configurations are aimed at, read from the sources."""
    gt = _src("graph_transformer.cu")
    ln = re.search(r"constexpr int kLnWidest = (\d+), kLnBackwardWidest = (\d+);", gt)
    assert ln, "kLnWidest / kLnBackwardWidest"
    row = re.search(r"#define HNH_DISPATCH_R\(r, CALL, FALLBACK\)(.*?)default:", _src("row_gather.cuh"), re.S)
    assert row, "HNH_DISPATCH_R"
    chunk = re.search(r"constexpr int64_t kMinChunkRows = (\d+);", _src("row_regs.cuh"))
    tn = re.search(r"constexpr int64_t kTnTargetCtas = (\d+), kTnMinChunk = (\d+);", _src("gat_kernels.cu"))
    assert chunk and tn, "kMinChunkRows / kTnMinChunk"
    # the register-row widths of pick_ln: r <= 64 kN for the kN of the table
    pick = re.search(r"K pick_ln\(int64_t r, (.*?)\) \{", _src("row_regs.cuh")).group(1)
    return dict(ln_widest=int(ln.group(1)), ln_backward_widest=int(ln.group(2)),
                attention=sorted(int(w) for w in re.findall(r"case (\d+):", row.group(1))),
                min_chunk_rows=int(chunk.group(1)), tn_min_chunk=int(tn.group(2)),
                ln_steps=sorted(int(k) for k in re.findall(r"K k(\d+)", pick) if int(k) > 0))


def paths(cfg, tables):
    """Per layer: the attention kernels ("fast" or "generic") and, with blocks, (LN forward, LN backward) ("regs" or
    "generic")."""
    att = tuple("fast" if d in tables["attention"] else "generic" for _, d, _ in cfg["layers"])
    if not cfg["ffn"]:
        return att, None
    side = lambda r, widest: "regs" if -(-r // 64) <= widest else "generic"  # noqa: E731
    return att, tuple((side(d * H, tables["ln_widest"]), side(d * H, tables["ln_backward_widest"])) for _, d, H in cfg["layers"])


@pytest.mark.parametrize("name", sorted(GT_CONFIGS))
def test_configurations_reach_their_paths(name):
    cfg, tables = GT_CONFIGS[name], kernel_tables()
    assert tables["ln_steps"][-1] >= tables["ln_widest"] >= tables["ln_backward_widest"]
    att, ln = paths(cfg, tables)
    assert att == tuple(cfg["attention"]), (name, "attention kernels", att, tables["attention"])
    assert ln == (tuple(tuple(x) for x in cfg["ln"]) if cfg["ln"] else None), (name, "LayerNorm tables", ln, tables)
    layers = cfg["layers"]
    widths = [d * H for _, d, H in layers]
    assert all(layers[l + 1][0] == widths[l] for l in range(len(layers) - 1))
    if name == "table":  # fast attention at d = 64 and 128, LN register rows at r = 256, FFN h = 512, everything on
        assert [d for _, d, _ in layers] == [64, 128] and widths == [256, 256] and cfg["ffn"] * widths[0] == 512
        assert cfg["edge_dim"] and cfg["beta"] and cfg["dropout"] > 0
    if name == "wide_heads":  # d = 256 and 8 heads of 32; ReLU between layers; no gate
        assert [(d, H) for _, d, H in layers] == [(256, 1), (32, 8)] and not cfg["ffn"] and not cfg["beta"]
    if name == "ln_backward_generic":  # just past the backward's register rows, inside the forward's
        assert (tables["ln_backward_widest"] * 64 < widths[0] <= (tables["ln_backward_widest"] + 1) * 64
                and cfg["edge_dim"] and cfg["beta"])
    if name == "ln_generic":
        assert tables["ln_widest"] * 64 < widths[0] <= (tables["ln_widest"] + 1) * 64
    if name == "odd":  # generic attention and one odd width: the scalar gate and LayerNorm paths
        assert any(r % 2 for r in widths) and cfg["edge_dim"] and cfg["beta"] and cfg["dropout"] > 0


@pytest.mark.parametrize("nproc", [1, 2, 4])
def test_the_skewed_graph_reaches_the_reduction_chunks_and_the_hub_row(nproc):
    """Row blocks of 4200 / p rows: more than one dw_chunks chunk on every rank, more than one TN split of k at p <= 4,
    a hub row of more than 2000 entries, and at p = 4 a third row block without entries."""
    tables = kernel_tables()
    rows_per_rank = -(-DEFAULT_N // nproc)
    assert rows_per_rank > tables["min_chunk_rows"] and rows_per_rank // tables["tn_min_chunk"] >= 2
    r, _ = (x.astype(np.int64) for x in skewed_tuples(DEFAULT_N, DEFAULT_N, 0xC0FFEE + 211))
    lens = np.bincount(r, minlength=DEFAULT_N)
    lm = landmarks(DEFAULT_N, DEFAULT_N)
    assert lens[lm["wide_hubs"][0]] > HUB_MIN > 2000
    if nproc == 4:
        assert lm["empty_rows"] == (2 * rows_per_rank, 3 * rows_per_rank) and not lens[2 * rows_per_rank:3 * rows_per_rank].any()
