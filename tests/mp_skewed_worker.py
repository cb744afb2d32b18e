"""Worker of the skewed-graph tests (tests/test_skewed_graphs_multirank_gpu.py launches it through
torch.distributed.run; tests/test_skewed_graphs_gpu.py calls run_case in-process at p = 1).  Per case every rank builds
the pattern of tests/skewed_graph.py, hands its round-robin share of the tuples to SpmatLocal.from_tuples, builds the
algorithm and runs the case's kind:

  base     the case's script of sddmmA/B, spmmA/B and fusedSpMM A/B on global A and B
  softmax  edge_softmax and edge_softmax_backward in both value orders, optionally with -inf scores
  attn     sparse_attention and sparse_attention_backward: plain, with dropout, with a per-head bias that masks, with
           edge features
  gat      GAT forward and backward with the case's attention kind
  train    GAT train steps
  gt       graph transformer forward and backward (a configuration of GT_CONFIGS)
  gt_train graph transformer node train steps
  gt_link  graph transformer link train steps against the targets of link_pairs, then link_evaluate
  gnn      PNA, GIN or GINE forward and backward (a configuration of GNN_CONFIGS)
  gnn_train  PNA, GIN or GINE node, link (the targets of link_pairs) or graph (readout_batch) train steps
  gine_int edge_relu_aggregate and its backward on integer inputs (exact results)
  max_agg  max_aggregate and its backward on inputs with exact ties
  distmult distmult_loss over T_pos = S (relations of distmult_relations) and T_neg (link_pairs), H_A = H_B
  rel_link GraphSAGE or R-GCN relational link train steps with the DistMult decoder, then relational_link_evaluate

GraphSAGE and R-GCN (SAGE_RGCN_CONFIGS) run as the gnn and gnn_train kinds.  S holds sval for base, the relations of
s_relations for R-GCN, those of distmult_relations for distmult, and ones otherwise.

Every op runs twice and the worker records whether the repeat gave the same bits.  It writes its rows of the results
-- or the error the layout must raise -- to <outdir>/<case>_rank<r>.npz.

Transports as in tests/mp_worker.py: "gloo" (ranks sharing one GPU), "nccl" (one GPU per rank)."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import gat_additive_oracle as gao  # noqa: E402
from tests import gin_oracle as go  # noqa: E402
from tests import graph_sage_oracle as gsa  # noqa: E402
from tests import graph_transformer_block_oracle as gbo  # noqa: E402
from tests import pna_oracle as po  # noqa: E402
from tests import rgcn_basis_oracle as bo  # noqa: E402
from tests import rgcn_oracle as ro  # noqa: E402
from tests.mp_edge_softmax_worker import score, upstream  # noqa: E402
from tests.mp_graph_transformer_worker import attr_of  # noqa: E402
from tests.mp_sparse_attention_edge_worker import edge_of  # noqa: E402
from tests.mp_worker import gather_local, sval  # noqa: E402
from tests.skewed_graph import DEFAULT_N, landmarks, rank_slice, skewed_tuples  # noqa: E402


def sizes(case):
    return case.get("m") or DEFAULT_N, case.get("n") or DEFAULT_N


def base_inputs(M, N, R, seed):
    """A (M x R) and B (N x R)."""
    rng = np.random.default_rng(seed + 11)
    return rng.uniform(-1, 1, (M, R)), rng.uniform(-1, 1, (N, R))


def attn_inputs(M, N, r, seed):
    """Q, dZ (M x r) and K, V (N x r)."""
    rng = np.random.default_rng(seed + 13)
    return rng.uniform(-1, 1, (M, r)), rng.uniform(-1, 1, (M, r)), rng.uniform(-1, 1, (N, r)), rng.uniform(-1, 1, (N, r))


def masked(rows, cols, M, N):
    """The entries a masking case scores -inf: every entry of the first wide hub row in the first of 4 column blocks
    (so one rank's share of that row is masked throughout while the others' is not), and in every fifth row every
    entry of an even column."""
    lm = landmarks(M, N)
    rows, cols = np.asarray(rows), np.asarray(cols)
    return ((rows == lm["wide_hubs"][0]) & (cols < lm["w"])) | ((rows % 5 == 1) & (cols % 2 == 0))


def bias_of(rows, cols, h, M, N):
    """b(u, v) of head h, a function of the global coordinates: up to +-30, -inf on masked(); head 1 also masks row 0
    throughout."""
    rows, cols = np.asarray(rows), np.asarray(cols)
    b = 30.0 * np.sin(0.37 * rows + 1.3 * cols + 0.5 * h)
    b[masked(rows, cols, M, N) | ((rows == 0) & (h == 1))] = -np.inf
    return b


def labels_of(N, classes, seed):
    """Labels on about 30 % of the nodes (40 % of the first three of 4 row blocks): every hub row labelled, the last
    row block unlabelled."""
    rng = np.random.default_rng(seed + 17)
    lm = landmarks(N, N)
    lab = rng.integers(0, classes, N)
    lab[rng.random(N) >= 0.4] = -1
    for u in (*lm["wide_hubs"], lm["last_block_hub"]):
        lab[u] = u % classes
    lab[lm["narrow_rows"][0]:] = -1
    return lab


def gat_inputs(N, layers, seed):
    """(X0, weights[layer][head], a1, a2, G) of a GAT case: weights scaled by 1 / sqrt(fan-in) so that the scores of a
    2000-entry row stay in exp's range."""
    rng = np.random.default_rng(seed + 19)
    X0 = rng.uniform(-1, 1, (N, layers[0][0]))
    ws = [[rng.uniform(-1, 1, (f, d)) / np.sqrt(f) for _ in range(H)] for f, d, H in layers]
    a1, a2 = gao.attention_inputs(layers, seed)
    G = rng.uniform(-1, 1, (N, layers[-1][1] * layers[-1][2]))
    return X0, ws, a1, a2, G


def coords_by_sddmm(alg, A, B, mode):
    """(row, col) of every entry of this rank's value vector of `mode` on any layout: SDDMMs of a global-index column
    against a column of ones (the column lives on the ranks whose submatrix starts at column 0)."""
    d = alg.dims
    like, sddmm = (alg.like_S_values, alg.sddmmA) if mode == "A" else (alg.like_ST_values, alg.sddmmB)
    ones, res = like(1.0), like(0.0)
    out = []
    for first in ("A", "B"):
        for m, which, shape in ((A, "A", (d.localArows, d.localAcols)), (B, "B", (d.localBrows, d.localBcols))):
            x = np.zeros(shape)
            flat, at = x.reshape(-1), 0
            for top, left, nr, nc in alg.submatrices(which):
                blk = np.zeros((nr, nc))
                if left == 0:
                    blk[:, 0] = np.arange(top, top + nr) if which == first else 1.0
                flat[at:at + nr * nc] = blk.reshape(-1)
                at += nr * nc
            m.from_host(x)
        alg.initial_shift(A, B, "sddmm" + mode)
        sddmm(A, B, ones, res)
        alg.de_shift(A, B, "sddmm" + mode)
        out.append(np.rint(res.to_host()).astype(np.int64))
    return out


def run_base(D, alg, case, M, N, out):
    d = alg.dims
    shapeA, shapeB = (d.localArows, d.localAcols), (d.localBrows, d.localBcols)
    subsA, subsB = alg.submatrices("A"), alg.submatrices("B")
    out.update(aSubmatrices=subsA, bSubmatrices=subsB, shapeA=shapeA, shapeB=shapeB)
    A, B = alg.like_A_matrix(), alg.like_B_matrix()
    vals, res = {}, {}
    for mode, like in (("A", alg.like_S_values), ("B", alg.like_ST_values)):
        r, c = coords_by_sddmm(alg, A, B, mode)
        out[f"{mode}_rows"], out[f"{mode}_cols"] = r, c
        vals[mode], res[mode] = like(0.0), like(0.0)
        vals[mode].from_host(sval(r, c))
    GA, GB = base_inputs(M, N, case["R"], case["seed"])
    hA, hB = gather_local(GA, subsA, shapeA), gather_local(GB, subsB, shapeB)
    for op in case["script"]:
        mode = op[-1]
        got = []
        for _ in range(2):
            A.from_host(hA)
            B.from_host(hB)
            res[mode].fill(0.0)
            shift = "spmm" + mode if op.startswith("spmm") else "sddmm" + mode
            alg.initial_shift(A, B, shift)
            if op.startswith("sddmm"):
                (alg.sddmmA if mode == "A" else alg.sddmmB)(A, B, vals[mode], res[mode])
            elif op.startswith("spmm"):
                (alg.spmmA if mode == "A" else alg.spmmB)(A, B, vals[mode])
            else:
                alg.fusedSpMM(A, B, vals[mode], res[mode], mode)
            alg.de_shift(A, B, shift)
            got.append(((A if mode == "A" else B).to_host(), res[mode].to_host()))
        out[op + "_repeat"] = all(np.array_equal(a, b, equal_nan=True) for a, b in zip(*got))
        if not op.startswith("sddmm"):
            out[op + "_dense"] = got[0][0]
        if not op.startswith("spmm"):
            out[op + "_values"] = got[0][1]


def run_softmax(D, alg, case, M, N, out):
    for mode in ("A", "B"):
        r, c = alg.entry_coordinates(mode)
        like = alg.like_S_values if mode == "A" else alg.like_ST_values
        x = score(r, c)
        if case.get("mask"):
            x[masked(r, c, M, N)] = -np.inf
        got = []
        for _ in range(2):
            v, g = like(0.0), like(0.0)
            v.from_host(x)
            alg.edge_softmax(v, mode)
            a = v.to_host()
            g.from_host(upstream(r, c))
            alg.edge_softmax_backward(v, g, mode)
            got.append((a, g.to_host()))
        out[f"{mode}_repeat"] = all(np.array_equal(a, b, equal_nan=True) for a, b in zip(*got))
        out.update({f"{mode}_rows": r, f"{mode}_cols": c, f"{mode}_alpha": got[0][0], f"{mode}_dx": got[0][1]})


def run_attn(D, alg, case, M, N, out):
    heads, d, variant, p = case["heads"], case["d"], case["variant"], case["dropout"]
    r = heads * d
    dims = alg.dims
    Q, K, V, dZ = alg.like_A_matrix(), alg.like_B_matrix(), alg.like_B_matrix(), alg.like_A_matrix()
    Z, dQ, dK, dV = alg.like_A_matrix(), alg.like_A_matrix(), alg.like_B_matrix(), alg.like_B_matrix()
    L = D.Dense.create(dims.localArows, heads)
    if case.get("rejected"):  # a layout without sparse attention must refuse before any launch
        alg.sparse_attention(Q, K, V, Z, L, heads)
        return
    Qg, dZg, Kg, Vg = attn_inputs(M, N, r, case["seed"])
    topA, _, nrA, _ = alg.submatrices("A")[0]
    topB, _, nrB, _ = alg.submatrices("B")[0]
    out.update(topA=topA, nrA=nrA, topB=topB, nrB=nrB)
    for m, g, top, nr in ((Q, Qg, topA, nrA), (dZ, dZg, topA, nrA), (K, Kg, topB, nrB), (V, Vg, topB, nrB)):
        m.from_host(gather_local(g, [(top, 0, nr, r)], m.shape))
    rA, cA = alg.entry_coordinates("A")
    rB, cB = alg.entry_coordinates("B")
    out.update(rA=rA, cA=cA, rB=rB, cB=cB)
    fwd, bwd, extra = dict(dropout=p, seed=case["mask_seed"]), {}, []
    if variant == "bias":
        vecs = []
        for rr, cc in ((rA, cA), (rB, cB)):
            b = np.concatenate([bias_of(rr, cc, h, M, N) for h in range(heads)])
            vecs.append(D.Vec.create(len(b)))
            vecs[-1].from_host(b)
        dbA, dbB = D.Vec.create(0), D.Vec.create(0)
        fwd.update(bias=vecs[0])
        bwd.update(bias_B=vecs[1], dbias=dbA, dbias_B=dbB)
        extra = [("dbA", dbA), ("dbB", dbB)]
    elif variant == "edge":
        edges = []
        for rr, cc in ((rA, cA), (rB, cB)):
            e = edge_of(rr, cc, r)
            edges.append(D.Dense.create(*e.shape))
            edges[-1].from_host(e)
        dE = D.Dense.create(1, 1)
        fwd.update(edge=edges[0])
        bwd.update(edge_B=edges[1], dedge=dE)
        extra = [("dE", dE)]
    got = []
    for _ in range(2):
        alg.sparse_attention(Q, K, V, Z, L, heads, **fwd)
        alg.sparse_attention_backward(Q, K, V, Z, L, dZ, dQ, dK, dV, heads, **fwd, **bwd)
        got.append({key: m.to_host() for key, m in [("Z", Z), ("L", L), ("dQ", dQ), ("dK", dK), ("dV", dV)] + extra})
    out["repeat"] = all(np.array_equal(got[0][k], got[1][k], equal_nan=True) for k in got[0])
    out.update(got[0])


def _gat(D, alg, case, N):
    layers = [tuple(l) for l in case["layers"]]
    X0, ws, a1, a2, G = gat_inputs(N, layers, case["seed"])
    net = D.GAT(alg, layers, 0.2, attention=case["attention"])
    if not case.get("rejected"):  # layouts that split R hold other weight shapes; they must refuse before reading them
        for l, (_, fph, H) in enumerate(layers):
            for h in range(H):
                net.set_weight(l, h, ws[l][h])
                if case["attention"] in ("additive", "gatv2"):
                    net.set_attention_vectors(l, h, a1[l][h], a2[l][h] if case["attention"] == "additive" else np.zeros(fph))
    return layers, X0, G, net


def run_gat(D, alg, case, M, N, out):
    layers, X0, G, net = _gat(D, alg, case, N)
    if case.get("rejected"):
        net.forward()
        return
    topA, _, nrA, _ = alg.submatrices("A")[0]
    topB, _, nrB, _ = alg.submatrices("B")[0]
    out.update(topA=topA, nrA=nrA, topB=topB, nrB=nrB)
    net.set_input(gather_local(X0, [(topB, 0, nrB, layers[0][0])], net.buffer_shape(0)))
    width = layers[-1][1] * layers[-1][2]
    Gl = gather_local(G, [(topA, 0, nrA, width)], net.buffer_shape(len(layers)))
    got = []
    for _ in range(2):
        net.forward()
        o = dict(out=net.buffer(len(layers)))
        net.backward(Gl)
        o["dX0"] = net.input_grad()
        for l, (_, _, H) in enumerate(layers):
            for h in range(H):
                o[f"dW_{l}_{h}"] = net.weight_grad(l, h)
                o[f"da1_{l}_{h}"], o[f"da2_{l}_{h}"] = net.attention_grads(l, h)
        got.append(o)
    out["repeat"] = all(np.array_equal(got[0][k], got[1][k], equal_nan=True) for k in got[0])
    out.update(got[0])


def run_train(D, alg, case, M, N, out):
    layers, X0, _, net = _gat(D, alg, case, N)
    topA = alg.submatrices("A")[0][0]
    topB, _, nrB, _ = alg.submatrices("B")[0]
    net.set_input(gather_local(X0, [(topB, 0, nrB, layers[0][0])], net.buffer_shape(0)))
    rows = net.buffer_shape(len(layers))[0]
    classes = layers[-1][1] * layers[-1][2]
    lab = -np.ones(rows, np.int64)
    hi = min(topA + rows, N)
    lab[:hi - topA] = labels_of(N, classes, case["seed"])[topA:hi]
    nl = D.NodeLabels(net, lab, classes)
    opt = D.AdamW(lr=1e-2)
    out["local_rows"] = rows
    out["steps"] = np.array([list(net.train_step(nl, opt)) for _ in range(case["steps"])])
    for l, (_, _, H) in enumerate(layers):
        for h in range(H):
            out[f"w{l}_{h}"] = net.weight(l, h)
            out[f"a1_{l}_{h}"], out[f"a2_{l}_{h}"] = net.attention_vectors(l, h)


# ---- the graph transformer -----------------------------------------------------------------------------------------
# Configurations and the paths each is meant to reach (tests/test_graph_transformer_sparse_oracle.py checks these
# against the kernels' tables): per layer the attention kernels ("fast": d in HNH_DISPATCH_R, else "generic") and,
# with blocks, LayerNorm forward and backward ("regs": the row in registers, else "generic").
GT_CONFIGS = {
    "table": dict(layers=[[64, 64, 4], [256, 128, 2]], edge_dim=3, beta=True, ffn=2, dropout=0.3,
                  attention=("fast", "fast"), ln=(("regs", "regs"), ("regs", "regs"))),
    "wide_heads": dict(layers=[[32, 256, 1], [256, 32, 8]], edge_dim=0, beta=False, ffn=0, dropout=0.0,
                       attention=("fast", "fast"), ln=None),
    "ln_backward_generic": dict(layers=[[48, 64, 17]], edge_dim=2, beta=True, ffn=1, dropout=0.3, attention=("fast",),
                                ln=(("regs", "generic"),)),
    "ln_generic": dict(layers=[[16, 64, 25]], edge_dim=0, beta=True, ffn=1, dropout=0.0, attention=("fast",),
                       ln=(("generic", "generic"),)),
    "odd": dict(layers=[[7, 5, 3], [15, 12, 2]], edge_dim=3, beta=True, ffn=1, dropout=0.3, attention=("generic", "generic"),
                ln=(("regs", "regs"), ("regs", "regs"))),
}


def gt_config(case):
    cfg = dict(GT_CONFIGS[case["gt"]])
    cfg["layers"] = [tuple(l) for l in cfg["layers"]]
    return cfg


def gt_inputs(N, cfg, seed):
    """(params, X, G) of a graph transformer case: the same on every rank."""
    layers = cfg["layers"]
    rng = np.random.default_rng(seed + 23)
    params = gbo.random_params(layers, cfg["edge_dim"], cfg["beta"], cfg["ffn"], rng)
    X = rng.uniform(-1, 1, (N, layers[0][0]))
    G = rng.uniform(-1, 1, (N, layers[-1][1] * layers[-1][2]))
    return params, X, G


def link_pairs(N, seed):
    """(rows, cols, soft targets) of the link cases' T: pairs on the wide hub rows, pairs between nodes without entries
    (the empty third row block), pairs into the hub column, random pairs, and duplicated pairs with equal targets."""
    rng = np.random.default_rng(seed + 29)
    lm = landmarks(N, N)
    e0, e1 = lm["empty_rows"]
    groups = [(np.full(40, u), rng.integers(0, N, 40)) for u in lm["wide_hubs"]]
    groups += [(rng.integers(e0, e1, 40), rng.integers(e0, e1, 40)), (rng.integers(0, N, 60), np.full(60, lm["hub_col"])),
               (rng.integers(0, N, 200), rng.integers(0, N, 200))]
    key = np.unique(np.concatenate([u * N + v for u, v in groups]))
    tr, tc = key // N, key % N
    y = rng.choice([0.0, 1.0, 0.25], len(tr))
    dup = rng.choice(len(tr), 6, replace=False)
    return np.concatenate([tr, tr[dup]]), np.concatenate([tc, tc[dup]]), np.concatenate([y, y[dup]])


def _gt(D, alg, case, N):
    cfg = gt_config(case)
    layers = cfg["layers"]
    net = D.GraphTransformer(alg, layers, edge_dim=cfg["edge_dim"], beta=cfg["beta"], ffn_ratio=cfg["ffn"])
    params, X, G = gt_inputs(N, cfg, case["seed"])
    for l, P in enumerate(params):
        for k, v in P.items():
            net.set_param(l, k, v)
    topA, _, nrA, _ = alg.submatrices("A")[0]
    topB, _, nrB, _ = alg.submatrices("B")[0]
    rA, cA = alg.entry_coordinates("A")
    rB, cB = alg.entry_coordinates("B")
    # what the case reached on this rank: local rows, entries in each value order, the longest A-order row
    reach = dict(topA=topA, nrA=nrA, topB=topB, nrB=nrB, local_rows=net.buffer_shape(0)[0], nA=len(rA), nB=len(rB),
                 longest=np.bincount(np.asarray(rA, np.int64)).max(initial=0) if len(rA) else 0)
    net.set_input(gather_local(X, [(topB, 0, nrB, layers[0][0])], net.buffer_shape(0)))
    if cfg["edge_dim"]:
        net.set_edge_attributes(attr_of(rA, cA, cfg["edge_dim"]), attr_of(rB, cB, cfg["edge_dim"]))
    return cfg, net, G, reach


def run_gt(D, alg, case, M, N, out):
    cfg, net, G, reach = _gt(D, alg, case, N)
    out.update(reach)
    layers = cfg["layers"]
    Gl = gather_local(G, [(reach["topA"], 0, reach["nrA"], G.shape[1])], net.buffer_shape(len(layers)))
    got = []
    for _ in range(2):
        net.forward(cfg["dropout"], case["mask_seed"])
        o = dict(Y=net.buffer(len(layers)))
        net.backward(Gl)
        o["dX"] = net.input_grad()
        for l in range(len(layers)):
            for k in net.param_names():
                o[f"g{l}_{k}"] = net.param_grad(l, k)
        got.append(o)
    out["repeat"] = all(np.array_equal(got[0][k], got[1][k], equal_nan=True) for k in got[0])
    out.update(got[0])


def _gt_params(net, layers, out):
    for l in range(len(layers)):
        for k in net.param_names():
            out[f"p{l}_{k}"] = net.param(l, k)


def run_gt_train(D, alg, case, M, N, out):
    cfg, net, _, reach = _gt(D, alg, case, N)
    out.update(reach)
    layers = cfg["layers"]
    rows = net.buffer_shape(len(layers))[0]
    classes = layers[-1][1] * layers[-1][2]
    topA = reach["topA"]
    lab = -np.ones(rows, np.int64)
    hi = min(topA + rows, N)
    lab[:hi - topA] = labels_of(N, classes, case["seed"])[topA:hi]
    nl = D.NodeLabels(net, lab, classes)
    opt = D.AdamW(lr=case["lrs"][0], weight_decay=0.01, max_grad_norm=case.get("clip"))
    steps = []
    for t, lr in enumerate(case["lrs"]):
        opt.lr = lr
        steps.append(list(net.train_step(nl, opt, cfg["dropout"], case["mask_seed"] + 7 * t)))
    out["steps"] = np.array(steps)
    _gt_params(net, layers, out)


def run_gt_link(D, alg, case, M, N, out):
    cfg, net, _, reach = _gt(D, alg, case, N)
    out.update(reach)
    layers = cfg["layers"]
    from distributed_sddmm_b200 import lib
    rank, world = lib().hnhd_world_rank(), lib().hnhd_world_size()
    tr, tc, y = link_pairs(N, case["seed"])
    sr, sc = rank_slice(tr, tc, rank, world)
    sy = y[rank::world]
    algT = D.Algorithm(case["alg"], D.SpmatLocal.from_tuples(N, N, sr.astype(np.uint64), sc.astype(np.uint64), sy), layers[0][0],
                       case["c"])
    t = D.LinkTargets(net, algT)
    opt = D.AdamW(lr=case["lrs"][0], weight_decay=0.01)
    steps = []
    for s, lr in enumerate(case["lrs"]):
        opt.lr = lr
        steps.append(list(net.link_train_step(t, opt, cfg["dropout"], case["mask_seed"] + 7 * s)))
    out["steps"] = np.array(steps)
    _gt_params(net, layers, out)
    loss, correct, count, scores = net.link_evaluate(t)
    out["evaluate"] = np.array([loss, correct, count])
    out["scores"] = scores
    out["tA_rows"], out["tA_cols"] = algT.entry_coordinates("A")
    out["H"] = net.buffer(len(layers))
    del t, algT


# ---- PNA, GIN and GINE ---------------------------------------------------------------------------------------------
# Configurations and, per layer, the width and the path of the layer's sparse aggregation (tests/test_skewed_gnn_fixture.py
# checks these against the kernels' tables): PNA gathers the statistics of z (input-wide) with multiAggregate, GIN sums
# X with spmmA, GINE sums ReLU(X_v + E_i) with edgeReluAggregate.  "table": one window of a width of HNH_DISPATCH_R
# (the 128-bit row kernels); "windows": wider than kWindow, so several column windows; "generic": an odd width, the
# one-warp-per-row kernels.
PNA_DEFAULT = (("mean", "min", "max", "std"), ("identity", "amplification", "attenuation"))
GNN_CONFIGS = {
    "pna_table": dict(model="pna", layers=[[64, 128], [128, 256], [256, 4]], aggregators=PNA_DEFAULT[0], scalers=PNA_DEFAULT[1],
                      reach=("table", "table", "table")),
    "pna_all": dict(model="pna", layers=[[128, 16], [16, 4]], aggregators=po.AGGREGATORS, scalers=po.SCALERS,
                    reach=("table", "table")),
    "pna_wide": dict(model="pna", layers=[[300, 4]], aggregators=("sum", "var"), scalers=("linear",), reach=("windows",)),
    "pna_odd": dict(model="pna", layers=[[7, 13], [13, 4]], aggregators=PNA_DEFAULT[0], scalers=PNA_DEFAULT[1],
                    reach=("generic", "generic")),
    "gin_table": dict(model="gin", layers=[[64, 32, 128], [128, 32, 256], [256, 32, 4]], edge_dim=0,
                      reach=("table", "table", "table")),
    "gine_table": dict(model="gin", layers=[[64, 32, 128], [128, 32, 256], [256, 32, 4]], edge_dim=3,
                       reach=("table", "table", "table")),
    "gine_odd": dict(model="gin", layers=[[7, 9, 13], [13, 9, 4]], edge_dim=2, reach=("generic", "generic")),
}
GINE_INT_WIDTH = 64  # the gine_int case: edge_relu_aggregate at a table width
TIE_ROWS = (4, 3154)  # rows without entries (row % 9 == 4) in the first and the last of 4 row blocks, given equal inputs
READOUT_GRAPHS, READOUT_CLASSES = 24, 3
GNN_LR = 1e-3  # the train cases: at 1e-2 the hub rows' sums make the losses grow tenfold per step


def gnn_config(case):
    cfg = dict(GNN_CONFIGS[case["gnn"]] if case["gnn"] in GNN_CONFIGS else SAGE_RGCN_CONFIGS[case["gnn"]])
    for k in ("aggr", "bases"):  # a case's own aggregation or basis count
        if k in case:
            cfg[k] = case[k]
    cfg["layers"] = [tuple(l) for l in cfg["layers"]]
    return cfg


_HIST = {}


def degree_histogram(N, seed):
    """The skewed graph's in-degree histogram (PNAConv's deg): the entries of each S-row, duplicates counted."""
    if (N, seed) not in _HIST:
        rows, _ = skewed_tuples(N, N, seed)
        _HIST[N, seed] = np.bincount(np.bincount(rows.astype(np.int64), minlength=N))
    return _HIST[N, seed]


def gnn_inputs(N, cfg, seed):
    """(params, X, G) of a PNA / GIN case, the same on every rank.  Rows TIE_ROWS of X are equal: they have no entries, so
    their outputs are equal too, which gives max readout a maximum attained on two ranks."""
    layers = cfg["layers"]
    rng = np.random.default_rng(seed + 37)
    if cfg["model"] == "pna":
        params = po.random_params(layers, len(cfg["aggregators"]), len(cfg["scalers"]), rng)
    elif cfg["model"] == "sage":
        params = gsa.random_params(layers, rng)
    elif cfg["model"] == "rgcn":
        params = bo.random_params(layers, NUM_RELATIONS, cfg["bases"], rng) if cfg.get("bases") else \
            ro.random_params(layers, NUM_RELATIONS, rng)
    else:
        params = go.random_params(layers, cfg["edge_dim"], rng)
    X = rng.uniform(-1, 1, (N, layers[0][0]))
    X[TIE_ROWS[1]] = X[TIE_ROWS[0]]
    G = rng.uniform(-1, 1, (N, layers[-1][-1]))
    return params, X, G


def gine_int_inputs(N, f, seed):
    """(X, dA) of the gine_int case: integers, so that X_v + E_i == 0 happens and every sum is exact."""
    rng = np.random.default_rng(seed + 43)
    return rng.integers(-3, 4, (N, f)).astype(np.float64), rng.integers(-3, 4, (N, f)).astype(np.float64)


def readout_batch(N, seed):
    """(batch, G, labels) of the graph train cases: graph 0 holds 150 random rows and hub row 3, so it spans every row
    block; graph 1 is TIE_ROWS alone (one maximum on two ranks); graph 2 is empty; the others take random rows; 10 % of
    the rows are in no graph; two graphs are unlabelled."""
    rng = np.random.default_rng(seed + 41)
    G = READOUT_GRAPHS
    batch = rng.integers(3, G, N)
    batch[rng.random(N) < 0.1] = -1
    batch[rng.choice(N, 150, replace=False)] = 0
    batch[landmarks(N, N)["wide_hubs"][0]] = 0
    batch[list(TIE_ROWS)] = 1
    labels = rng.integers(0, READOUT_CLASSES, G)
    labels[[5, 9]] = -1
    return batch, G, labels


def readout_head(width, seed):
    rng = np.random.default_rng(seed + 47)
    return rng.uniform(-1, 1, (width, READOUT_CLASSES)), rng.uniform(-0.5, 0.5, READOUT_CLASSES)


def _gnn(D, alg, case, N):
    cfg = gnn_config(case)
    layers = cfg["layers"]
    if cfg["model"] == "pna":
        net = D.PNA(alg, layers, aggregators=cfg["aggregators"], scalers=cfg["scalers"], deg=degree_histogram(N, case["seed"]))
    elif cfg["model"] == "sage":
        net = D.GraphSAGE(alg, layers, aggr=cfg["aggr"])
    elif cfg["model"] == "rgcn":
        net = D.RGCN(alg, layers, num_relations=NUM_RELATIONS, aggr=cfg["aggr"], num_bases=cfg.get("bases"))
    else:
        net = D.GIN(alg, layers, edge_dim=cfg["edge_dim"], eps=0.0, train_eps=case.get("train_eps", True))
    params, X, G = gnn_inputs(N, cfg, case["seed"])
    for l, P in enumerate(params):
        for k, v in P.items():
            net.set_param(l, k, v)
    topA, _, nrA, _ = alg.submatrices("A")[0]
    topB, _, nrB, _ = alg.submatrices("B")[0]
    rA, cA = alg.entry_coordinates("A")
    rB, cB = alg.entry_coordinates("B")
    # what the case reached on this rank: local rows, entries in each value order, the longest A-order row
    reach = dict(topA=topA, nrA=nrA, topB=topB, nrB=nrB, local_rows=net.buffer_shape(0)[0], nA=len(rA), nB=len(rB),
                 longest=np.bincount(np.asarray(rA, np.int64)).max(initial=0) if len(rA) else 0)
    net.set_input(gather_local(X, [(topB, 0, nrB, layers[0][0])], net.buffer_shape(0)))
    if cfg["model"] == "gin" and cfg["edge_dim"]:
        net.set_edge_attributes(go.attr_of(rA, cA, cfg["edge_dim"]), go.attr_of(rB, cB, cfg["edge_dim"]))
    return cfg, net, G, reach


def _gnn_params(net, layers, out):
    for l in range(len(layers)):
        for k in net.param_names():
            out[f"p{l}_{k}"] = net.param(l, k)


def run_gnn(D, alg, case, M, N, out):
    cfg, net, G, reach = _gnn(D, alg, case, N)
    out.update(reach)
    layers = cfg["layers"]
    Gl = gather_local(G, [(reach["topA"], 0, reach["nrA"], G.shape[1])], net.buffer_shape(len(layers)))
    got = []
    for _ in range(2):
        net.forward()
        o = dict(Y=net.buffer(len(layers)))
        net.backward(Gl)
        o["dX"] = net.input_grad()
        for l in range(len(layers)):
            for k in net.param_names():
                o[f"g{l}_{k}"] = net.param_grad(l, k)
        got.append(o)
    out["repeat"] = all(np.array_equal(got[0][k], got[1][k], equal_nan=True) for k in got[0])
    out.update(got[0])


def run_gnn_train(D, alg, case, M, N, out):
    """Three node, link or graph train steps (case["task"])."""
    cfg, net, _, reach = _gnn(D, alg, case, N)
    out.update(reach)
    layers = cfg["layers"]
    rows = net.buffer_shape(len(layers))[0]
    topA = reach["topA"]
    hi = min(topA + rows, N)
    opt = D.AdamW(lr=GNN_LR)
    if case["task"] == "node":
        lab = -np.ones(rows, np.int64)
        lab[:hi - topA] = labels_of(N, layers[-1][-1], case["seed"])[topA:hi]
        nl = D.NodeLabels(net, lab, layers[-1][-1])
        out["steps"] = np.array([list(net.train_step(nl, opt)) for _ in range(case["steps"])])
    elif case["task"] == "link":
        from distributed_sddmm_b200 import lib
        rank, world = lib().hnhd_world_rank(), lib().hnhd_world_size()
        tr, tc, y = link_pairs(N, case["seed"])
        sr, sc = rank_slice(tr, tc, rank, world)
        algT = D.Algorithm(case["alg"], D.SpmatLocal.from_tuples(N, N, sr.astype(np.uint64), sc.astype(np.uint64), y[rank::world]),
                           layers[0][0], case["c"])
        t = D.LinkTargets(net, algT)
        out["steps"] = np.array([list(net.link_train_step(t, opt)) for _ in range(case["steps"])])
        del t, algT
    else:
        batch, G, labels = readout_batch(N, case["seed"])
        local = np.full(rows, -1, np.int64)
        local[:hi - topA] = batch[topA:hi]
        ro = D.GraphReadout(net, local, G, pool=case["pool"], num_classes=READOUT_CLASSES)
        W_head, b_head = readout_head(layers[-1][-1], case["seed"])
        ro.set_param("weight", W_head)
        ro.set_param("bias", b_head)
        gl = D.GraphLabels(ro, labels, READOUT_CLASSES)
        out["steps"] = np.array([list(net.graph_train_step(ro, gl, opt)) for _ in range(case["steps"])])
        for k in ro.param_names():
            out[f"head_{k}"] = ro.param(k)
        del gl, ro
    _gnn_params(net, layers, out)


# ---- GraphSAGE, R-GCN and DistMult ---------------------------------------------------------------------------------
# Configurations as GNN_CONFIGS': GraphSAGE aggregates X (mean and sum with spmmA, max with maxAggregate), R-GCN X per
# relation (relationalAggregate) or per basis (basisAggregate), each at its layer's input width.  "aggr" is the default
# a case may override; the *_link configurations feed the DistMult decoder at their output width.
SAGE_RGCN_CONFIGS = {
    "sage_table": dict(model="sage", aggr="max", layers=[[64, 128], [128, 256], [256, 4]], reach=("table", "table", "table")),
    "sage_wide": dict(model="sage", aggr="max", layers=[[300, 4]], reach=("windows",)),
    "sage_odd": dict(model="sage", aggr="max", layers=[[7, 13], [13, 4]], reach=("generic", "generic")),
    "rgcn_table": dict(model="rgcn", aggr="mean", layers=[[64, 128], [128, 256], [256, 4]], reach=("table", "table", "table")),
    "rgcn_wide": dict(model="rgcn", aggr="mean", layers=[[300, 4]], reach=("windows",)),
    "rgcn_odd": dict(model="rgcn", aggr="mean", layers=[[7, 13], [13, 4]], reach=("generic", "generic")),
    "basis_table": dict(model="rgcn", aggr="mean", bases=3, layers=[[64, 128], [128, 256], [256, 4]],
                        reach=("table", "table", "table")),
    "basis_many": dict(model="rgcn", aggr="mean", bases=30, layers=[[64, 4]], reach=("table",)),  # more bases than registers
    "rgcn_link": dict(model="rgcn", aggr="mean", layers=[[64, 128], [128, 64]], reach=("table", "table")),
    "sage_link": dict(model="sage", aggr="max", layers=[[64, 128], [128, 256]], reach=("table", "table")),
}
# R-GCN's S and DistMult's targets declare one relation more than their relations use: relation 5 is carried by no entry
NUM_RELATIONS, USED_RELATIONS = 6, 5
MAX_AGG_WIDTHS = (64, 128, 256, 300, 7)
DISTMULT_WIDTHS = (64, 128, 256, 7, 300)


def copies(rows, cols, N):
    """Per tuple, how many earlier copies of its pair the list holds."""
    keys = np.asarray(rows, np.int64) * N + np.asarray(cols, np.int64)
    o = np.argsort(keys, kind="stable")
    ks = keys[o]
    start = np.r_[0, np.flatnonzero(ks[1:] != ks[:-1]) + 1]
    out = np.empty(len(ks), np.int64)
    out[o] = np.arange(len(ks)) - np.repeat(start, np.diff(np.r_[start, len(ks)]))
    return out


def s_relations(rows, cols, N):
    """R-GCN's relation of every tuple of S's global list (rgcn_oracle.hashed_relations: the copies of a duplicate
    differ).  A rank takes its slice of these: hashed on the rank's own slice, a copy would lose its earlier copies."""
    return ro.hashed_relations(rows, cols, N, USED_RELATIONS)


def distmult_relations(rows, cols, N):
    """DistMult's relation of every tuple of a target list: relation 0 for the wide hub rows and a third of the rest, so
    that it spans more than 8 pieces of HNH_EDGE_PIECE at p = 1 and more than one on every rank at p = 4; the others
    hashed over 1 .. 4; the k-th copy of a pair moves k relations on, so copies differ."""
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    base = np.where(np.isin(rows, landmarks(N, N)["wide_hubs"]) | ((rows * 31 + cols * 17) % 3 == 0), 0,
                    1 + (rows * 7 + cols * 3) % 4)
    return ((base + copies(rows, cols, N)) % USED_RELATIONS).astype(np.float64)


def distmult_targets(N, seed):
    """(T_pos, T_neg) as (rows, cols, relations): the skewed graph's own tuples, and link_pairs' pairs."""
    pr, pc = (x.astype(np.int64) for x in skewed_tuples(N, N, seed))
    nr, nc, _ = link_pairs(N, seed)
    return (pr, pc, distmult_relations(pr, pc, N)), (nr, nc, distmult_relations(nr, nc, N))


def distmult_inputs(N, r, seed):
    """(H, relation table) of the distmult case."""
    rng = np.random.default_rng(seed + 53)
    return rng.uniform(-1, 1, (N, r)), rng.uniform(-1, 1, (NUM_RELATIONS, r))


def max_agg_inputs(N, f, seed):
    """(X, dZ) of the max_agg case: X >= 0 with about half its entries exactly 0 (ties), rows TIE_ROWS equal."""
    rng = np.random.default_rng(seed + 59)
    X = np.maximum(rng.standard_normal((N, f)), 0.0)
    X[TIE_ROWS[1]] = X[TIE_ROWS[0]]
    return X, rng.standard_normal((N, f))


def run_max_agg(D, alg, case, M, N, out):
    """max_aggregate and its backward at width case["R"]."""
    f = case["R"]
    X, dZh = max_agg_inputs(N, f, case["seed"])
    topA, _, nrA, _ = alg.submatrices("A")[0]
    topB, _, nrB, _ = alg.submatrices("B")[0]
    nA, nB = alg.like_A_matrix().shape[0], alg.like_B_matrix().shape[0]
    Xd, Z, Cn, dZ, dX = (D.Dense.create(n, f) for n in (nB, nA, nA, nA, nB))
    Xd.from_host(gather_local(X, [(topB, 0, nrB, f)], (nB, f)))
    dZ.from_host(gather_local(dZh, [(topA, 0, nrA, f)], (nA, f)))
    rA, _ = alg.entry_coordinates("A")
    out.update(topA=topA, nrA=nrA, topB=topB, nrB=nrB, nA=len(rA),
               longest=np.bincount(np.asarray(rA, np.int64)).max(initial=0) if len(rA) else 0)
    got = []
    for _ in range(2):
        alg.max_aggregate(Xd, Z, Cn)
        alg.max_aggregate_backward(Xd, Z, Cn, dZ, dX)
        got.append(dict(Z=Z.to_host(), C=Cn.to_host(), dX=dX.to_host()))
    out["repeat"] = all(np.array_equal(got[0][k], got[1][k]) for k in got[0])
    out.update(got[0])


def _rank_targets(D, case, N, trip, width):
    """An Algorithm over this rank's round-robin share of the triples trip = (rows, cols, relations)."""
    from distributed_sddmm_b200 import lib
    rank, world = lib().hnhd_world_rank(), lib().hnhd_world_size()
    sr, sc = rank_slice(trip[0].astype(np.uint64), trip[1].astype(np.uint64), rank, world)
    return D.Algorithm(case["alg"], D.SpmatLocal.from_tuples(N, N, sr, sc, trip[2][rank::world].copy()), width, case["c"])


def run_distmult(D, alg, case, M, N, out):
    """distmult_loss at r = case["R"] with H_A = H_B: S is T_pos; a positive call and an accumulated negative call over
    T_neg, twice."""
    r = case["R"]
    pos, neg = distmult_targets(N, case["seed"])
    algN = _rank_targets(D, case, N, neg, r)
    H, rel = distmult_inputs(N, r, case["seed"])
    topA, _, nrA, _ = alg.submatrices("A")[0]
    Hl = D.Dense.create(alg.like_A_matrix().shape[0], r)
    Hl.from_host(gather_local(H, [(topA, 0, nrA, r)], Hl.shape))
    Dd = D.Dense.create(NUM_RELATIONS, r)
    Dd.from_host(rel)
    dH, dD = D.Dense.create(*Hl.shape), D.Dense.create(NUM_RELATIONS, r)
    sp, sn = alg.like_S_values(), algN.like_S_values()
    inv = 1.0 / (len(pos[0]) + len(neg[0]))
    erp, ecp = alg.entry_coordinates("A")
    ern, ecn = algN.entry_coordinates("A")
    out.update(topA=topA, nrA=nrA, nA=len(erp), erp=erp, ecp=ecp, ern=ern, ecn=ecn)
    got = []
    for _ in range(2):
        res = [alg.distmult_loss(Hl, Hl, Dd, NUM_RELATIONS, 1.0, inv, dH, dH, dD, sp),
               algN.distmult_loss(Hl, Hl, Dd, NUM_RELATIONS, 0.0, inv, dH, dH, dD, sn, accumulate=True)]
        got.append(dict(res=np.array(res, np.float64), dH=dH.to_host(), dD=dD.to_host(), sp=sp.to_host(), sn=sn.to_host()))
    out["repeat"] = all(np.array_equal(got[0][k], got[1][k]) for k in got[0])
    out.update(got[0])
    del algN


def run_rel_link(D, alg, case, M, N, out):
    """Relational link train steps of a GraphSAGE or R-GCN configuration with the DistMult decoder over
    distmult_targets, then relational_link_evaluate."""
    cfg, net, _, reach = _gnn(D, alg, case, N)
    out.update(reach)
    layers = cfg["layers"]
    pos, neg = distmult_targets(N, case["seed"])
    algP, algN = _rank_targets(D, case, N, pos, layers[0][0]), _rank_targets(D, case, N, neg, layers[0][0])
    dec = D.DistMultDecoder(net, NUM_RELATIONS)
    dec.set_param("rel", distmult_inputs(N, layers[-1][-1], case["seed"])[1])
    t = D.RelationalLinkTargets(net, algP, algN, NUM_RELATIONS)
    opt = D.AdamW(lr=GNN_LR)
    out["steps"] = np.array([list(net.relational_link_train_step(dec, t, opt)) for _ in range(case["steps"])])
    out["rel"], out["drel"] = dec.param("rel"), dec.param_grad("rel")
    _gnn_params(net, layers, out)
    loss, correct, count, sp, sn = net.relational_link_evaluate(dec, t)
    out["evaluate"] = np.array([loss, correct, count])
    out["sp"], out["sn"] = sp, sn
    out["erp"], out["ecp"] = algP.entry_coordinates("A")
    out["ern"], out["ecn"] = algN.entry_coordinates("A")
    out["H"] = net.buffer(len(layers))
    del t, dec, algP, algN


def run_gine_int(D, alg, case, M, N, out):
    """edge_relu_aggregate and its backward on integer X, dA and E = gin_oracle.edge_rows: every partial sum is an
    integer far below 2^53, so the results are exact."""
    f = case["R"]
    X, dA = gine_int_inputs(N, f, case["seed"])
    topA, _, nrA, _ = alg.submatrices("A")[0]
    topB, _, nrB, _ = alg.submatrices("B")[0]
    nA, nB = alg.like_A_matrix().shape[0], alg.like_B_matrix().shape[0]
    Xd, A, dAd, dX, dE = D.Dense.create(nB, f), D.Dense.create(nA, f), D.Dense.create(nA, f), D.Dense.create(nB, f), D.Dense.create(0, 0)
    rA, cA = alg.entry_coordinates("A")
    rB, cB = alg.entry_coordinates("B")
    EA, EB = D.Dense.create(len(rA), f), D.Dense.create(len(rB), f)
    if len(rA):
        EA.from_host(go.edge_rows(rA, cA, f))
    if len(rB):
        EB.from_host(go.edge_rows(rB, cB, f))
    Xd.from_host(gather_local(X, [(topB, 0, nrB, f)], (nB, f)))
    dAd.from_host(gather_local(dA, [(topA, 0, nrA, f)], (nA, f)))
    out.update(topA=topA, nrA=nrA, topB=topB, nrB=nrB, rA=rA, cA=cA, nA=len(rA))
    got = []
    for _ in range(2):
        alg.edge_relu_aggregate(Xd, EA, A)
        alg.edge_relu_aggregate_backward(Xd, EA, EB, dAd, dX, dE)
        got.append(dict(A=A.to_host(), dX=dX.to_host(), dE=dE.to_host()))
    out["repeat"] = all(np.array_equal(got[0][k], got[1][k]) for k in got[0])
    out.update(got[0])


KINDS = dict(base=run_base, softmax=run_softmax, attn=run_attn, gat=run_gat, train=run_train, gt=run_gt, gt_train=run_gt_train,
             gt_link=run_gt_link, gnn=run_gnn, gnn_train=run_gnn_train, gine_int=run_gine_int, max_agg=run_max_agg,
             distmult=run_distmult, rel_link=run_rel_link)


def s_values(case, rows, cols, tr, tc, rank, world):
    """The values of this rank's tuples tr, tc: slices of what the global list rows, cols defines."""
    N = sizes(case)[1]
    if case["kind"] == "base":
        return sval(tr, tc)
    if case["kind"] == "distmult":
        return distmult_relations(rows, cols, N)[rank::world].copy()
    if case.get("gnn") and gnn_config(case)["model"] == "rgcn":
        return s_relations(rows, cols, N)[rank::world].copy()
    return np.ones(len(tr))


def run_case(D, case, rank, world):
    """The case on this rank: {key: array}, with "error" = the message if the library refused."""
    M, N = sizes(case)
    rows, cols = skewed_tuples(M, N, case["seed"])
    tr, tc = rank_slice(rows, cols, rank, world)
    S = D.SpmatLocal.from_tuples(M, N, tr, tc, s_values(case, rows, cols, tr, tc, rank, world))
    alg = D.Algorithm(case["alg"], S, case["R"], case["c"])
    out = {}
    try:
        KINDS[case["kind"]](D, alg, case, M, N, out)
    except RuntimeError as e:
        out["error"] = str(e)
        if not case.get("rejected"):  # shown by the launcher if the other ranks then wait for this one
            print(f"rank {rank}: {case['name']}: {e}", flush=True)
    del alg, S
    return out


def main():
    cases = json.loads(sys.argv[1])
    outdir = sys.argv[2]
    transport = sys.argv[3]
    import torch
    ngpu = torch.cuda.device_count()
    if ngpu:
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")) % ngpu if transport == "nccl" else 0)
    from distributed_sddmm_b200 import driver as D
    rank, world = D.world_init(transport)
    for case in cases:
        if rank == 0:  # progress, shown when the launcher reports a failure or a timeout
            print("case", case["name"], flush=True)
        np.savez(os.path.join(outdir, f"{case['name']}_rank{rank}.npz"), **run_case(D, case, rank, world))
    D.world_finalize()


if __name__ == "__main__":
    main()
