"""The GraphSAGE, R-GCN and DistMult cases of the skewed-graph tests (mp_skewed_worker.SAGE_RGCN_CONFIGS and the
max_agg, distmult and rel_link cases), checked without a GPU: that they reach the kernels they are aimed at, and that
no pass can be decided by a floating-point tie or threshold.

  * Every configuration aggregates at the widths it names, by HNH_DISPATCH_R and kWindow as graph_sage.cu and rgcn.cu
    state them (R-GCN's row kernels also need an even f); the op cases' widths reach the table, window and generic
    paths; DistMult's r > 256 goes to the kS = 0 generic kernels.
  * In every max aggregation of the fp64 model (every layer of every max configuration, and the max readout over
    readout_batch) each neighbour either equals the maximum exactly or lies below it by more than 1e-9 of its column's
    scale, and exact ties at 0 (ReLU zeros) are split over several column blocks.
  * No ReLU pre-activation that is not exactly 0 lies within 1e-12 of 0 at its column's scale; no DistMult score of the
    op cases lies within 1e-9 of 0 at the scores' scale.
  * The relations: relation 0 of T_pos spans more than 8 pieces, and more than one in every row and column block with
    entries; copies of a pair carry different relations in S and in both target lists; relation 5 is carried by none."""
import re

import numpy as np
import pytest
import torch

from tests import distmult_oracle as dmo
from tests import graph_sage_oracle as gsa
from tests import mp_skewed_worker as W
from tests.skewed_graph import PIECE, landmarks
from tests.test_skewed_gnn_fixture import _src, graph, path
from tests.test_skewed_graphs_multirank_gpu import SAGE_RGCN_OTHER, SAGE_RGCN_TABLE, SEED, s_relations, sage_rgcn_model

SAGE_MAX = [name for name, cfg in W.SAGE_RGCN_CONFIGS.items() if cfg["model"] == "sage" and cfg["aggr"] == "max"]
MODELS = sorted({(name, tuple(sorted(kw.items()))) for name, kw in SAGE_RGCN_TABLE + SAGE_RGCN_OTHER}
                | {(name, ()) for name in ("rgcn_link", "sage_link")} | {("rgcn_link", (("bases", 3),))})


def tables():
    """(HNH_DISPATCH_R's widths, the column window of graph_sage.cu and rgcn.cu, DistMult's widest register path)."""
    row = re.search(r"#define HNH_DISPATCH_R\(r, CALL, FALLBACK\)(.*?)default:", _src("row_gather.cuh"), re.S)
    assert row, "HNH_DISPATCH_R"
    windows = [re.search(r"constexpr int kWindow = (\d+);", _src(f)) for f in ("graph_sage.cu", "rgcn.cu")]
    assert all(windows) and windows[0].group(1) == windows[1].group(1), "kWindow"
    # R-GCN's row kernels take an even f only
    assert len(re.findall(r"table_width\(w\)[^{]*f % 2 == 0\)", _src("rgcn.cu"))) == 4, "rgcn.cu's f % 2 == 0"
    wide = re.search(r"r <= (\d+) \? distmult_bce_generic_kernel<8> : distmult_bce_generic_kernel<0>", _src("distmult.cu"))
    assert wide, "distmult.cu's kS = 0 kernel"
    return sorted(int(w) for w in re.findall(r"case (\d+):", row.group(1))), int(windows[0].group(1)), int(wide.group(1))


def rgcn_path(f, table, window):
    return "generic" if f <= window and f % 2 else path(f, table, window)


@pytest.mark.parametrize("name", sorted(W.SAGE_RGCN_CONFIGS))
def test_configurations_reach_their_aggregation_paths(name):
    table, window, _ = tables()
    cfg = W.SAGE_RGCN_CONFIGS[name]
    widths = [l[0] for l in cfg["layers"]]  # both models aggregate their layer input
    reach = rgcn_path if cfg["model"] == "rgcn" else path
    got = tuple(reach(w, table, window) for w in widths)
    assert got == tuple(cfg["reach"]), (name, "aggregates at", widths, "reaching", got, "not", cfg["reach"], table, window)
    layers = cfg["layers"]
    assert all(layers[l + 1][0] == layers[l][-1] for l in range(len(layers) - 1)), name
    if name.endswith("_table"):
        assert widths == [w for w in table if w >= 64], (name, widths, table)
    if name.endswith("_wide"):
        assert widths[0] > window and widths[0] % window
    if name.endswith("_odd"):
        assert all(w % 2 for w in widths), name
    if name == "basis_many":  # more bases than the row kernel at f = 64 (G = 32 lanes) keeps in registers
        acc = re.search(r"constexpr int kBasisAcc = (\d+);", _src("rgcn.cu"))
        assert acc and widths == [64] and cfg["bases"] > int(acc.group(1)) // (64 // 32), name
    if name.endswith("_link"):  # the DistMult decoder at its table widths
        assert path(layers[-1][-1], table, window) == "table"


def test_op_cases_reach_every_path():
    table, window, wide = tables()
    assert {path(f, table, window) for f in W.MAX_AGG_WIDTHS} == {"table", "windows", "generic"}
    assert [f for f in W.MAX_AGG_WIDTHS if path(f, table, window) == "table"] == [w for w in table if w >= 64]
    assert [f for f in W.DISTMULT_WIDTHS if f in table] == [w for w in table if w >= 64]
    assert any(f > wide for f in W.DISTMULT_WIDTHS) and any(f not in table and f <= 32 for f in W.DISTMULT_WIDTHS)


def _model(name, kw):
    """(rows, cols, N, cfg, params, X) of a configuration."""
    N, rows, cols = graph()
    cfg = W.gnn_config(dict(gnn=name, **dict(kw)))
    params, X, _ = W.gnn_inputs(N, cfg, SEED)
    return rows, cols, N, cfg, params, X


def _layers(name, kw):
    """Per layer (input, pre-activation) of the fp64 model."""
    rows, cols, N, cfg, params, X = _model(name, kw)
    rels = s_relations(dict(seed=SEED)) if cfg["model"] == "rgcn" else None
    out, h = [], gsa._t(X)
    with torch.no_grad():
        for l, P in enumerate(params):
            one = dict(cfg, layers=[cfg["layers"][l]])
            y = sage_rgcn_model(one, rows, cols, rels, N)([{k: gsa._t(v) for k, v in P.items()}], h)
            out.append((h.numpy(), y.numpy()))
            h = torch.relu(y)
    return out


def _no_close_max(rows, cols, M, X, where):
    """Every neighbour equals the column's maximum over its row exactly or lies below it by more than 1e-9 of the
    column's scale; returns the (row, column) cells whose maximum is an exact tie at 0."""
    Z, C = gsa.max_aggregate(rows, cols, M, X)
    scale = np.abs(X).max(0)
    gap = Z[rows] - X[cols]
    assert ((gap == 0) | (gap > 1e-9 * scale)).all(), (where, int(((gap != 0) & (gap <= 1e-9 * scale)).sum()))
    return (Z == 0) & (C >= 2)


@pytest.mark.parametrize("name", SAGE_MAX)
def test_no_max_is_decided_by_rounding(name):
    """Every max layer of the configuration; beyond the first layer (inputs after a ReLU) exact ties at 0 spread over
    more than one of the 4 column blocks of the row, so that ranks split dZ / C between them, and both copies of a
    duplicate attain a maximum somewhere."""
    N, rows, cols = graph()
    lm = landmarks(N, N)
    dup = np.flatnonzero(np.diff(rows * N + cols) == 0)
    for l, (h, _) in enumerate(_layers(name, {})):
        ties = _no_close_max(rows, cols, N, h, (name, l))
        Z, _ = gsa.max_aggregate(rows, cols, N, h)
        assert (h[cols[dup]] == Z[rows[dup]]).any(), (name, l, "no duplicate attains a maximum")
        if l > 0:
            u, k = np.nonzero(ties)
            spread = [len(np.unique(cols[(rows == uu) & (h[cols, kk] == 0)] // lm["w"])) for uu, kk in zip(u[:200], k[:200])]
            assert len(u) > 100 and max(spread) > 1, (name, l, len(u))


def test_no_max_readout_is_decided_by_rounding():
    """The max readout over readout_batch of sage_table's output: graph 1 (TIE_ROWS) ties exactly, nothing else is close."""
    rows, cols, N, cfg, params, X = _model("sage_table", {})
    with torch.no_grad():
        Y = sage_rgcn_model(cfg, rows, cols, None, N)([{k: gsa._t(v) for k, v in P.items()} for P in params], gsa._t(X)).numpy()
    batch, G, _ = W.readout_batch(N, SEED)
    keep = batch >= 0
    ties = _no_close_max(batch[keep], np.flatnonzero(keep), G, Y, "readout")
    assert ties.sum() == 0 and np.array_equal(Y[W.TIE_ROWS[0]], Y[W.TIE_ROWS[1]])


@pytest.mark.parametrize("name,kw", MODELS, ids=lambda x: x if isinstance(x, str) else "_".join(f"{k}{v}" for k, v in x))
def test_no_relu_is_decided_by_rounding(name, kw):
    for l, (_, y) in enumerate(_layers(name, kw)[:-1]):
        scale = np.abs(y).max(0)
        near = (y != 0) & (np.abs(y) <= 1e-12 * scale)
        assert not near.any() and (y < 0).any() and (y > 0).any(), (name, kw, l, int(near.sum()))


@pytest.mark.parametrize("r", W.DISTMULT_WIDTHS)
def test_no_distmult_score_is_near_zero(r):
    N = graph()[0]
    pos, neg = W.distmult_targets(N, SEED)
    H, rel = (dmo._t(x) for x in W.distmult_inputs(N, r, SEED))
    s = torch.cat([dmo.scores(H, H, rel, *pos)[0], dmo.scores(H, H, rel, *neg)[0]]).numpy()
    assert (np.abs(s) > 1e-9 * np.abs(s).max()).all() and (s > 0).any() and (s < 0).any(), r


def _copies_differ(rows, cols, rels, N):
    keys = rows * N + cols
    o = np.lexsort((rels, keys))
    k, v = keys[o], rels[o]
    same = np.flatnonzero(k[1:] == k[:-1])
    return len(same) and not (v[same] == v[same + 1]).any()


def test_relations_hold_what_the_cases_need():
    N, rows, cols = graph()
    lm = landmarks(N, N)
    (pr, pc, prel), (nr, nc, nrel) = W.distmult_targets(N, SEED)
    srel = s_relations(dict(seed=SEED))
    U = W.USED_RELATIONS
    assert W.NUM_RELATIONS == U + 1
    for r_, c_, v in ((rows, cols, srel), (pr, pc, prel), (nr, nc, nrel)):
        assert np.array_equal(np.unique(v), np.arange(U)), "every relation but the last is carried"
        assert _copies_differ(r_, c_, v, N), "copies of a pair carry different relations"
    # S's relations come from the global list: hashed per rank slice, a copy would repeat an earlier copy's relation
    assert np.array_equal(np.sort(pr * N + pc), np.sort(rows * N + cols))
    zero = prel == 0
    assert zero.sum() > 8 * PIECE, "relation 0 spans more than one piece per warp of the dD sum"
    q = lm["q"]
    for keys in (pr, pc):  # the row and the column blocks of 4 ranks
        for b in range(4):
            held = keys // q == b
            assert not held.any() or (zero & held).sum() > PIECE, (b, (zero & held).sum())
    assert not (pr // q == 2).any()  # the empty row block: no T_pos entry
    assert (nrel == 0).any() and np.isin(nr, lm["wide_hubs"]).any()
