"""The distributed ops on a skewed graph (tests/skewed_graph.py: hub rows of more than two softmax pieces spread over
every rank's column block, a hub column, a rank whose row block is empty, a column band nothing touches, duplicates and
self-loops, 4200 nodes so that 4 ranks hold 1050 rows each) at the kernels' table widths, on 1, 2 and 4 ranks
(tests/mp_skewed_worker.py): the base ops at R = 64, 128, 256 and 100 on every layout, the edge softmax with and without
-inf scores, fused sparse attention (plain, dropout, a masking per-head bias, edge features) at heads x d = 2 x 64,
1 x 128 and 4 x 7, GAT forward and backward with the four attention kinds and GAT train steps, and the graph
transformer (the configurations of mp_skewed_worker.GT_CONFIGS: forward and backward, node and link train steps,
link_evaluate), and PNA, GIN and GINE (the configurations of mp_skewed_worker.GNN_CONFIGS, aggregating at 64, 128
and 256, past one 256-wide column window and at odd widths: forward and backward, node, link and graph train steps with
all three pools, and GINE's edge-ReLU aggregation on integers, exact), GraphSAGE and R-GCN with and without bases (the
configurations of mp_skewed_worker.SAGE_RGCN_CONFIGS, at the same widths: forward and backward, node, link, graph and
relational link train steps), max_aggregate and distmult_loss at 64, 128, 256, 300 and 7, each against the fp64
models written per stored entry, rank by rank.  Beyond parity: rows without entries give Z = 0, L = -inf and zero dQ, and PNA's and GIN's
output from the row's own input alone; untouched columns zero dK, dV and GINE's dX; a repeat gives the same bits; the
results at p = 2 and 4 equal those at p = 1 to 1e-12; per-entry gradients (dbias, dE) of the two copies of a duplicate
agree, with dropout too (one keep bit per (row, column), whatever the layout); parameter gradients and trained
parameters are bit-identical across ranks; GINE on 15d_fusion2 at p = 4 has a rank without A-order entries; the
relation no entry carries gets exactly 0 in R-GCN's weight or comp gradient and in DistMult's dD, and DistMult's
correct count matches exactly.

One worker launch per rank count serves every test of that count.  Ranks share cuda:0 over the gloo-backed transport
unless there is one GPU per rank (then NCCL)."""
import json
import math
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from tests import gat_additive_oracle as gao
from tests import gat_backward_oracle as gbk
from tests import gat_softmax_oracle as gso
from tests import gatv2_oracle as gv2
from tests import distmult_oracle as dmo
from tests import gin_oracle as go
from tests import graph_readout_oracle as gro
from tests import graph_sage_oracle as gsa
from tests import graph_transformer_sparse_oracle as gts
from tests import link_prediction_oracle as lpo
from tests import mp_skewed_worker as W
from tests import pna_oracle as po
from tests import rgcn_basis_oracle as bo
from tests import rgcn_oracle as ro
from tests import sparse_attention_bias_oracle as sb
from tests import sparse_attention_dropout_oracle as sd
from tests import sparse_attention_edge_oracle as se
from tests import sparse_attention_oracle as sa
from tests import training_oracle as tro
from tests.mp_edge_softmax_worker import score, upstream
from tests.mp_graph_transformer_worker import attr_of
from tests.mp_sparse_attention_edge_worker import edge_of
from tests.mp_util import ROOT, free_port
from tests.mp_worker import gather_local, sval
from tests.skewed_graph import PIECE, landmarks, skewed_tuples
from tests.test_distmult_multirank_gpu import _scores_match
from tests.test_graph_transformer_gpu import grad_err
from tests.test_graph_transformer_sparse_oracle import kernel_tables, paths as gt_paths
from tests.test_sparse_attention_multirank_gpu import rel_err

pytestmark = pytest.mark.gpu
SEED = 0xC0FFEE + 211
GAT_LAYERS = [[64, 32, 2], [64, 16, 4]]  # per-head products at table widths 32 and 16 from inputs 64 wide
# widths per layout: every layout sees table widths inside its shift loops, the dense-shift layouts the generic kernels too
BASE_WIDTHS = {"15d_fusion1": [64, 128, 256, 100], "15d_fusion2": [128, 100], "15d_sparse": [256, 128],
               "25d_dense_replicate": [256, 128], "25d_sparse_replicate": [64, 128]}
REPLICATION = {1: {a: [1] for a in BASE_WIDTHS},
               2: {"15d_fusion1": [1, 2], "15d_fusion2": [1, 2], "15d_sparse": [1, 2], "25d_sparse_replicate": [2]},
               4: {"15d_fusion1": [1, 2], "15d_fusion2": [1, 2], "15d_sparse": [1, 2], "25d_dense_replicate": [1],
                   "25d_sparse_replicate": [1]}}
ALL_OPS = ["sddmmA", "spmmA", "spmmB", "fusedA", "sddmmB", "fusedB"]


def _case(kind, alg, c, R, **kw):
    tag = "_".join(f"{k}{v}" for k, v in sorted(kw.items()) if k not in ("layers", "script", "mask_seed", "steps", "lrs"))
    return dict(name=f"{kind}_{alg}_c{c}_R{R}" + ("_" + tag if tag else ""), kind=kind, alg=alg, c=c, R=R, seed=SEED, **kw)


GT_CLIP = 1.0  # below the first step's gradient norm of the "table" train case (3.6), above the later ones (about 0.5)


def gt_case(kind, alg, c, config, **kw):
    """A graph transformer case of configuration `config` (mp_skewed_worker.GT_CONFIGS)."""
    return _case(kind, alg, c, W.GT_CONFIGS[config]["layers"][0][0], gt=config, mask_seed=31, **kw)


def gnn_case(kind, alg, c, config, **kw):
    """A PNA, GIN, GINE, GraphSAGE or R-GCN case of configuration `config` (mp_skewed_worker.GNN_CONFIGS or
    SAGE_RGCN_CONFIGS)."""
    return _case(kind, alg, c, W.gnn_config(dict(gnn=config))["layers"][0][0], gnn=config, **kw)


# GraphSAGE and R-GCN forward and backward: (configuration, case keywords); the table ones on every full-row layout
SAGE_RGCN_TABLE = [("sage_table", dict(aggr=a)) for a in ("mean", "sum", "max")] + \
    [("rgcn_table", dict(aggr=a)) for a in ("mean", "sum")] + [("basis_table", {})]
SAGE_RGCN_OTHER = [(name, {}) for name in ("sage_wide", "sage_odd", "rgcn_wide", "rgcn_odd", "basis_many")]
TABLE_WIDTHS = (64, 128, 256)


def cases_for(p):
    out = []
    for alg, cs in REPLICATION[p].items():
        for i, R in enumerate(BASE_WIDTHS[alg]):
            c = cs[i % len(cs)]
            # local kernel fusion with c > 1 accumulates its fused output onto the gathered operand: not what the global
            # model states, and covered against the reference's own code in tests/test_multirank_gpu.py
            script = [op for op in ALL_OPS if not (alg == "15d_fusion2" and c > 1 and op.startswith("fused"))]
            out.append(_case("base", alg, c, R, script=script))
    c2 = 2 if p > 1 else 1  # replication needs at least 2 ranks
    out += [_case("softmax", "15d_fusion1", 1, 8), _case("softmax", "15d_fusion1", c2, 8, mask=1),
            _case("softmax", "15d_fusion2", 1, 8), _case("softmax", "15d_fusion1", 1, 8, mask=1)]

    def attn(alg, c, heads, d, variant, dropout=0.0):
        return _case("attn", alg, c, heads * d, heads=heads, d=d, variant=variant, dropout=dropout, mask_seed=29)

    out += [attn("15d_fusion1", 1, 2, 64, "plain"), attn("15d_fusion2", 1, 1, 128, "plain"), attn("15d_fusion1", c2, 4, 7, "plain"),
            attn("15d_fusion1", 1, 1, 128, "plain", 0.4), attn("15d_fusion2", 1, 2, 64, "plain", 0.4),
            attn("15d_fusion1", 1, 2, 64, "bias", 0.4), attn("15d_fusion2", 1, 4, 7, "bias"),
            attn("15d_fusion1", c2, 1, 128, "bias"),
            attn("15d_fusion1", 1, 1, 128, "edge"), attn("15d_fusion1", c2, 2, 64, "edge", 0.4),
            attn("15d_fusion2", 1, 4, 7, "edge")]
    for kind, alg, c in (("leaky", "15d_fusion1", 1), ("softmax", "15d_fusion2", 1), ("additive", "15d_fusion1", c2),
                         ("gatv2", "15d_fusion1", 1)):
        out.append(_case("gat", alg, c, 64, attention=kind, layers=GAT_LAYERS))
    out += [_case("train", "15d_fusion1", 1, 64, attention="additive", layers=GAT_LAYERS, steps=3),
            _case("train", "15d_fusion2", 1, 64, attention="softmax", layers=GAT_LAYERS, steps=3)]
    out += [gt_case("gt", alg, c, name) for name in ("table", "odd") for alg, c in (("15d_fusion1", 1), ("15d_fusion1", c2),
                                                                                     ("15d_fusion2", 1))]
    if p == 4:  # rank 2's row block holds no entries (see check_gt_reach)
        out.append(gt_case("gt", "15d_fusion1", 1, "ln_backward_generic"))
    out += [gt_case("gt_train", "15d_fusion1", 1, "table", lrs=[1e-2, 3e-2, 2e-2], clip=GT_CLIP),
            gt_case("gt_train", "15d_fusion1", 1, "wide_heads", lrs=[1e-2] * 3),
            gt_case("gt_link", "15d_fusion1", 1, "table", lrs=[1e-2, 2e-2, 1e-2])]
    # PNA, GIN and GINE: every configuration on the three layouts with full rows, the op on integers, and train steps
    gnn_layouts = (("15d_fusion1", 1), ("15d_fusion1", c2), ("15d_fusion2", 1))
    out += [gnn_case("gnn", alg, c, name) for name in W.GNN_CONFIGS for alg, c in gnn_layouts]
    out += [gnn_case("gnn", "15d_fusion1", 1, "gin_table", train_eps=False)]
    out += [_case("gine_int", alg, c, W.GINE_INT_WIDTH) for alg, c in gnn_layouts]
    out += [gnn_case("gnn_train", "15d_fusion1", 1, name, task="node", steps=3, **kw)
            for name, kw in (("pna_table", {}), ("gin_table", {}), ("gin_table", dict(train_eps=False)), ("gine_table", {}))]
    out += [gnn_case("gnn_train", "15d_fusion1", 1, name, task="link", steps=3) for name in ("pna_table", "gine_table")]
    out += [gnn_case("gnn_train", "15d_fusion1", 1, name, task="graph", pool=pool, steps=3)
            for name in ("pna_table", "gin_table") for pool in gro.POOLS]
    # GraphSAGE, R-GCN and DistMult: the table widths on the three layouts with full rows, the others on 15d_fusion1
    out += [gnn_case("gnn", alg, c, name, **kw) for name, kw in SAGE_RGCN_TABLE for alg, c in gnn_layouts]
    out += [gnn_case("gnn", "15d_fusion1", 1, name, **kw) for name, kw in SAGE_RGCN_OTHER]
    for kind, widths in (("max_agg", W.MAX_AGG_WIDTHS), ("distmult", W.DISTMULT_WIDTHS)):
        out += [_case(kind, alg, c, f) for f in widths for alg, c in (gnn_layouts if f in TABLE_WIDTHS else gnn_layouts[:1])]
    out += [gnn_case("gnn_train", "15d_fusion1", 1, name, task="node", steps=3, aggr=a)
            for name, a in (("sage_table", "max"), ("rgcn_table", "mean"), ("basis_table", "sum"))]
    out += [gnn_case("gnn_train", "15d_fusion1", 1, name, task="link", steps=3, aggr=a)
            for name, a in (("sage_table", "max"), ("rgcn_table", "mean"))]
    out += [gnn_case("gnn_train", "15d_fusion1", 1, name, task="graph", pool=pool, steps=3, aggr=a)
            for name, a, pool in (("sage_table", "max", "max"), ("sage_table", "max", "mean"), ("rgcn_table", "mean", "sum"))]
    out += [gnn_case("rel_link", "15d_fusion1", 1, name, steps=3, **kw)
            for name, kw in (("rgcn_link", {}), ("rgcn_link", dict(bases=3)), ("sage_link", {}))]
    if p > 1:  # the layouts that split R have no row softmax, attention, GAT backward, graph transformer, PNA or GIN
        out += [dict(attn("15d_sparse", 1, 2, 64, "plain"), rejected=1),
                dict(_case("gat", "15d_sparse", 1, 64, attention="softmax", layers=GAT_LAYERS), rejected=1),
                dict(gt_case("gt", "15d_sparse", 1, "table"), rejected=1), dict(gt_case("gt", "15d_fusion2", 2, "odd"), rejected=1)]
        out += [dict(gnn_case("gnn", alg, c, name), rejected=1) for name in ("pna_table", "gine_table")
                for alg, c in (("15d_sparse", 1), ("15d_fusion2", 2))]
        out += [dict(gnn_case("gnn", alg, c, name, **kw), rejected=1) for name, kw in SAGE_RGCN_TABLE
                for alg, c in (("15d_sparse", 1), ("15d_fusion2", 2))]
        out += [dict(_case("distmult", alg, c, 64), rejected=1) for alg, c in (("15d_sparse", 1), ("15d_fusion2", 2))]
    return list({c["name"]: c for c in out}.values())  # at p = 1 the c = 2 cases fall onto their c = 1 twins


CASES = {p: cases_for(p) for p in (1, 2, 4)}


def params(kind, ps=(1, 2, 4), **match):
    return [pytest.param(p, c, id=f"p{p}-{c['name']}") for p in ps for c in CASES[p]
            if c["kind"] == kind and not c.get("rejected") and all(c.get(k) == v for k, v in match.items())]


_RESULTS = {}


def results(nproc, timeout=2400):
    """{case name: [per-rank dict]} of every case of this rank count: one launch, kept for the module."""
    if nproc in _RESULTS:
        return _RESULTS[nproc]
    cases = CASES[nproc]
    transport = "self" if nproc == 1 else "nccl" if torch.cuda.device_count() >= nproc else "gloo"
    with tempfile.TemporaryDirectory() as td:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
               "--master-addr", "127.0.0.1", "--master-port", str(free_port()),
               os.path.join(ROOT, "tests", "mp_skewed_worker.py"), json.dumps(cases), td, transport]
        env = dict(os.environ, OMP_NUM_THREADS="2")
        p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=timeout, text=True)
        if p.returncode != 0 and "Address already in use" in p.stdout:  # lost the race for the rendezvous port
            cmd[cmd.index("--master-port") + 1] = str(free_port())
            p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=timeout, text=True)
        assert p.returncode == 0, "worker failed:\n" + p.stdout[-6000:]
        out = {}
        for c in cases:
            out[c["name"]] = []
            for r in range(nproc):
                z = np.load(os.path.join(td, f"{c['name']}_rank{r}.npz"), allow_pickle=False)
                out[c["name"]].append({k: z[k] for k in z.files})
    _RESULTS[nproc] = out
    return out


_GRAPH = {}


def graph(case):
    """(M, N, rows, cols) of a case as int64, sorted by (row, col) with the duplicates kept."""
    M, N = W.sizes(case)
    if (M, N) not in _GRAPH:
        r, c = (x.astype(np.int64) for x in skewed_tuples(M, N, case["seed"]))
        order = np.lexsort((c, r))
        _GRAPH[M, N] = (r[order], c[order])
    return (M, N, *_GRAPH[M, N])


def lookup(N, rows, cols, values, qr, qc):
    """values (one per stored entry of the sorted rows, cols) at the entries (qr, qc); the copies of a duplicate are
    equal in every per-entry model (inputs that are functions of (row, col)), so the first copy stands for all."""
    key = rows * N + cols
    at = np.searchsorted(key, qr * N + qc)
    assert np.array_equal(key[at], qr * N + qc)
    return values[at]


def ranks_ok(ranks, name):
    for r, d in enumerate(ranks):
        assert "error" not in d, (name, r, str(d.get("error")))
    return ranks


def assemble(ranks, key, top, nr, total):
    """The global matrix from every rank's rows [top, top + nr) of `key`; all rows must be covered."""
    first = ranks[0][key]
    G = np.full((total,) + first.shape[1:], np.nan)
    covered = np.zeros(total, bool)
    for d in ranks:
        t, n = int(d[top]), min(int(d[nr]), total - int(d[top]))
        G[t:t + n] = d[key][:n]
        covered[t:t + n] = True
    assert covered.all(), key
    return G


def check_rows(ranks, name, key, want, top, nr, tol=1e-10):
    """Every rank's rows of `key` against the model's, +-inf matched exactly; returns the assembled global matrix."""
    total = len(want)
    for r, d in enumerate(ranks):
        t, n = int(d[top]), min(int(d[nr]), total - int(d[top]))
        got, w = d[key][:n], want[t:t + n]
        fin = np.isfinite(w)
        assert np.array_equal(fin, np.isfinite(got)) and np.array_equal(got[~fin], w[~fin]), (name, r, key)
        err = np.abs(got[fin] - w[fin]).max(initial=0.0) / max(np.abs(want[np.isfinite(want)]).max(initial=0.0), 1e-300)
        assert err < tol, (name, r, key, err)
    return assemble(ranks, key, top, nr, total)


# ---- base ops ------------------------------------------------------------------------------------------------------
_BASE_REF = {}


def base_reference(case, ones):
    """Dense results of the global model for the case's width: S's value at (u, v) is sval(u, v) per stored copy (ones:
    1 per copy), so duplicates add up, as in the scipy matrix of oracle.hnh_oracle.global_reference."""
    import scipy.sparse as sp
    M, N, rows, cols = graph(case)
    key = (M, N, case["R"], ones)
    if key not in _BASE_REF:
        A, B = W.base_inputs(M, N, case["R"], case["seed"])
        v = np.ones(len(rows)) if ones else sval(rows, cols)
        S = sp.csr_matrix((v, (rows, cols)), shape=(M, N))  # sums the copies of a duplicate
        ri = np.repeat(np.arange(M), np.diff(S.indptr))
        Sd = sp.csr_matrix((S.data * np.einsum("ij,ij->i", A[ri], B[S.indices]), S.indices, S.indptr), shape=(M, N))
        _BASE_REF[key] = dict(spmmA=S @ B, spmmB=S.T @ A, fusedA=Sd @ B, fusedB=Sd.T @ A)
    return _BASE_REF[key]


def check_base(ranks, case, nproc):
    ranks = ranks_ok(ranks, case["name"])
    M, N, rows, cols = graph(case)
    A, B = W.base_inputs(M, N, case["R"], case["seed"])
    for mode in ("A", "B"):  # every stored pair is held by some rank, in both value orders
        keys = np.concatenate([d[f"{mode}_rows"] * N + d[f"{mode}_cols"] for d in ranks])
        assert np.array_equal(np.unique(keys), np.unique(rows * N + cols)), (case["name"], mode)
        if case["c"] == 1 and not case["alg"].startswith("25d"):
            assert np.array_equal(np.sort(keys), rows * N + cols), (case["name"], mode, "copies of duplicates")
    for op in case["script"]:
        mode = op[-1]
        # local kernel fusion treats S as an all-ones pattern and leaves the SDDMM buffer unfilled
        ones = case["alg"] == "15d_fusion2" and op.startswith("fused")
        for r, d in enumerate(ranks):
            where = (case["name"], op, r)
            assert bool(d[op + "_repeat"]), where
            if not op.startswith("spmm") and not ones:
                u, v = d[f"{mode}_rows"], d[f"{mode}_cols"]
                want = sval(u, v) * np.einsum("ij,ij->i", A[u], B[v])
                assert np.abs(d[op + "_values"] - want).max(initial=0.0) <= 1e-10 * np.abs(want).max(initial=1e-300), where
            if not op.startswith("sddmm"):
                G = base_reference(case, ones)[op]
                subs, shape = (d["aSubmatrices"], d["shapeA"]) if mode == "A" else (d["bSubmatrices"], d["shapeB"])
                want = gather_local(G, [tuple(int(x) for x in s) for s in subs], tuple(int(x) for x in shape))
                assert np.abs(d[op + "_dense"] - want).max() <= 1e-10 * np.abs(G).max(), where


# ---- edge softmax --------------------------------------------------------------------------------------------------
def check_softmax(ranks, case, nproc):
    ranks = ranks_ok(ranks, case["name"])
    M, N, rows, cols = graph(case)
    x = score(rows, cols)
    if case.get("mask"):
        x[W.masked(rows, cols, M, N)] = -np.inf
    alpha = gso.edge_softmax_np(x, rows, M)
    # a row masked throughout is NaN, as torch.softmax gives (fused sparse attention defines Z = 0, L = -inf there)
    dx = gso.edge_softmax_backward_np(alpha, upstream(rows, cols), rows, M)
    hub = landmarks(M, N)["wide_hubs"][0]
    for mode in ("A", "B"):
        keys = []
        for r, d in enumerate(ranks):
            where = (case["name"], mode, r)
            assert bool(d[f"{mode}_repeat"]), where
            u, v = d[f"{mode}_rows"], d[f"{mode}_cols"]
            for got, w in ((d[f"{mode}_alpha"], lookup(N, rows, cols, alpha, u, v)), (d[f"{mode}_dx"], lookup(N, rows, cols, dx, u, v))):
                nan = np.isnan(w)
                assert np.array_equal(np.isnan(got), nan) and nan.sum() <= 0.01 * len(nan), where
                assert rel_err(got[~nan], w[~nan]) < 1e-13, where
            keys.append(u * N + v)
        assert np.array_equal(np.sort(np.concatenate(keys)), rows * N + cols), (case["name"], mode)  # duplicates included
        assert (rows == hub).sum() > 2 * 1024 + 37  # the hub row is more than two pieces long


# ---- fused sparse attention ----------------------------------------------------------------------------------------
_ATTN_REF = {}


def attention_reference(case):
    """The model's Z, L, dQ, dK, dV and per-entry gradients for a case (the same at every rank count)."""
    key = (W.sizes(case), case["heads"], case["d"], case["variant"], case["dropout"])
    if key in _ATTN_REF:
        return _ATTN_REF[key]
    M, N, rows, cols = graph(case)
    heads, d, p, seed = case["heads"], case["d"], case["dropout"], case["mask_seed"]
    Q, dZ, K, V = W.attn_inputs(M, N, heads * d, case["seed"])
    scale = 1 / math.sqrt(d)
    want = {}
    if case["variant"] == "plain" and p == 0.0:
        want["Z"], want["L"] = sa.forward_np(rows, cols, M, Q, K, V, heads, scale)
        want["dQ"], want["dK"], want["dV"] = sa.backward_np(rows, cols, M, Q, K, V, dZ, heads, scale)
    elif case["variant"] == "plain":
        want["Z"], want["L"] = sd.forward_np(rows, cols, M, Q, K, V, heads, scale, p, seed)
        want["dQ"], want["dK"], want["dV"] = sd.backward_np(rows, cols, M, Q, K, V, dZ, heads, scale, p, seed)
    elif case["variant"] == "bias":
        bias = np.concatenate([W.bias_of(rows, cols, h, M, N) for h in range(heads)])
        want["Z"], want["L"] = sb.forward_np(rows, cols, M, Q, K, V, bias, heads, scale, p, seed)
        want["dQ"], want["dK"], want["dV"], want["db"] = sb.backward_np(rows, cols, M, Q, K, V, dZ, bias, heads, scale, p, seed)
    else:
        E = edge_of(rows, cols, heads * d)
        want["Z"], want["L"] = se.forward_np(rows, cols, M, Q, K, V, E, heads, scale, p, seed)
        want["dQ"], want["dK"], want["dV"], want["dE"], _ = se.backward_np(rows, cols, M, Q, K, V, E, dZ, heads, scale, p, seed)
    _ATTN_REF[key] = want
    return want


def check_attention(ranks, case, nproc):
    name = case["name"]
    ranks = ranks_ok(ranks, name)
    M, N, rows, cols = graph(case)
    want = attention_reference(case)
    heads = case["heads"]
    for r, d in enumerate(ranks):
        assert bool(d["repeat"]), (name, r)
    got = {}
    for key in ("Z", "L", "dQ"):
        got[key] = check_rows(ranks, name, key, want[key], "topA", "nrA")
    for key in ("dK", "dV"):
        got[key] = check_rows(ranks, name, key, want[key], "topB", "nrB")
    # rows without entries, and the columns nothing points to
    empty = np.bincount(rows, minlength=M) == 0
    lm = landmarks(M, N)
    assert empty[lm["empty_rows"][0]:lm["empty_rows"][1]].all() and empty.mean() > 0.25
    assert not got["Z"][empty].any() and np.isneginf(got["L"][empty]).all() and not got["dQ"][empty].any(), name
    untouched = np.bincount(cols, minlength=N) == 0
    assert untouched[lm["empty_cols"][0]:lm["empty_cols"][1]].all()
    assert not got["dK"][untouched].any() and not got["dV"][untouched].any(), name
    if case["variant"] == "bias" and heads > 1:
        assert np.isneginf(want["L"][0, 1]) and np.isfinite(want["L"][0, 0])  # row 0 is masked throughout in head 1 only
    # per-entry gradients, matched by (row, col): the copies of a duplicate agree (with dropout: they share one keep bit)
    nnz = len(rows)
    dup = np.flatnonzero(np.diff(rows * N + cols) == 0)
    assert len(dup) >= 50 and (rows[dup] == lm["dup_row"]).sum() >= 3
    for r, d in enumerate(ranks):
        if case["variant"] == "bias":
            for order, u, v in (("dbA", d["rA"], d["cA"]), ("dbB", d["rB"], d["cB"])):
                n = len(u)
                assert d[order].shape == (heads * n,), (name, r, order)
                for h in range(heads):
                    w = lookup(N, rows, cols, want["db"][h * nnz:(h + 1) * nnz], u, v)
                    assert rel_err(d[order][h * n:(h + 1) * n], w) < 1e-10, (name, r, order, h)
        if case["variant"] == "edge":
            assert rel_err(d["dE"], lookup(N, rows, cols, want["dE"], d["rA"], d["cA"])) < 1e-10, (name, r, "dE")
    if case["dropout"] > 0 and case["variant"] != "plain":
        # the dropped entries show as rows of dE (or entries of dbias) that lose their D w alpha dZ term: what the model
        # computes from the hash of the global (row, col) is what every layout computes, copy by copy
        key, u, v = ("dE", "rA", "cA") if case["variant"] == "edge" else ("dbA", "rA", "cA")
        allk = np.concatenate([d[u] * N + d[v] for d in ranks])
        vals = np.concatenate([d[key] if key == "dE" else d[key][:len(d[u])] for d in ranks])
        order = np.argsort(allk, kind="stable")
        allk, vals = allk[order], vals[order]
        same = np.flatnonzero(np.diff(allk) == 0)
        assert len(same) >= 50 and np.array_equal(vals[same], vals[same + 1]), (name, "copies of a duplicate differ")


# ---- GAT -----------------------------------------------------------------------------------------------------------
def gat_forward(kind, ri, ci, N, layers, ws, u1, u2, x):
    if kind == "leaky":
        return gbk.gat_forward_torch(ri, ci, N, layers, ws, 0.2, x)
    if kind == "softmax":
        return gso.gat_softmax_forward_torch(ri, ci, N, layers, ws, 0.2, x)
    if kind == "additive":
        return gao.gat_additive_forward_torch(ri, ci, N, layers, ws, u1, u2, 0.2, x)
    return gv2.gatv2_forward_torch(ri, ci, N, layers, ws, u1, 0.2, x)


def gat_tensors(case, grad=True):
    """The case's inputs as torch leaves, and the stored entries with their duplicates (the models' edges() would
    merge them; the forward functions take any edge list)."""
    M, N, rows, cols = graph(case)
    layers = [tuple(l) for l in case["layers"]]
    X0, ws, a1, a2, G = W.gat_inputs(N, layers, case["seed"])
    t = lambda v: torch.tensor(np.asarray(v, np.float64), requires_grad=grad)  # noqa: E731
    nest = lambda n: [[t(v) for v in l] for l in n]  # noqa: E731
    return N, layers, torch.from_numpy(rows), torch.from_numpy(cols), t(X0), nest(ws), nest(a1), nest(a2), G


_GAT_REF = {}


def gat_reference(case):
    if case["attention"] not in _GAT_REF:
        N, layers, ri, ci, x, ws, u1, u2, G = gat_tensors(case)
        out = gat_forward(case["attention"], ri, ci, N, layers, ws, u1, u2, x)
        out.backward(torch.from_numpy(G))
        g = lambda v: v.grad.numpy() if v.grad is not None else np.zeros(v.shape)  # noqa: E731
        want = dict(out=out.detach().numpy(), dX0=g(x))
        for l, (_, _, H) in enumerate(layers):
            for h in range(H):
                want[f"dW_{l}_{h}"] = g(ws[l][h])
                if case["attention"] in ("additive", "gatv2"):
                    want[f"da1_{l}_{h}"] = g(u1[l][h])
                if case["attention"] == "additive":
                    want[f"da2_{l}_{h}"] = g(u2[l][h])
        _GAT_REF[case["attention"]] = want
    return _GAT_REF[case["attention"]]


def check_gat(ranks, case, nproc):
    name = case["name"]
    ranks = ranks_ok(ranks, name)
    want = gat_reference(case)
    assert np.abs(want["out"]).max() > 0 and np.abs(want["dX0"]).max() > 0
    for r, d in enumerate(ranks):
        assert bool(d["repeat"]), (name, r)
    check_rows(ranks, name, "out", want["out"], "topA", "nrA")
    check_rows(ranks, name, "dX0", want["dX0"], "topB", "nrB")
    for key, w in want.items():
        if key[0] == "d" and key != "dX0":
            assert np.abs(w).max() > 0, (name, key)
            for r, d in enumerate(ranks):
                assert np.array_equal(d[key], ranks[0][key]), (name, r, key, "differs across ranks")
            assert rel_err(ranks[0][key], w) < 1e-10, (name, key)


def check_training(ranks, case, nproc):
    """3 train steps: the cross-entropy and the parameter-gradient reductions run over 1050 local rows at p = 4 (more
    than two row chunks of 512), with one rank's row block unlabelled and another's without entries."""
    name = case["name"]
    ranks = ranks_ok(ranks, name)
    if nproc == 4:
        assert all(int(d["local_rows"]) >= 2 * 512 + 1 for d in ranks)
    for r, d in enumerate(ranks):
        for k in d:
            assert np.array_equal(d[k], ranks[0][k]), (name, r, k, "differs across ranks")
    N, layers, ri, ci, x, ws, u1, u2, _ = gat_tensors(case)
    x = x.detach()
    labels = W.labels_of(N, layers[-1][1] * layers[-1][2], case["seed"])
    lm = landmarks(N, N)
    assert 0.2 < (labels >= 0).mean() < 0.4 and (labels[lm["narrow_rows"][0]:] < 0).all() and labels[lm["wide_hubs"][0]] >= 0
    leaves = [w for l in ws for w in l]
    if case["attention"] == "additive":
        leaves += [v for l1, l2 in zip(u1, u2) for v in l1 + l2]
    res = tro.train(lambda _: gat_forward(case["attention"], ri, ci, N, layers, ws, u1, u2, x), leaves, labels, case["steps"],
                    lr=1e-2)
    steps = ranks[0]["steps"]
    for t, w in enumerate(res):
        assert abs(steps[t][0] - w[0]) <= 1e-10 * abs(w[0]) and abs(steps[t][3] - w[3]) <= 1e-10 * abs(w[3]), (name, t)
        assert (int(steps[t][1]), int(steps[t][2])) == (w[1], w[2]), (name, t)
    for l, (_, _, H) in enumerate(layers):
        for h in range(H):
            read = [(f"a1_{l}_{h}", u1[l][h]), (f"a2_{l}_{h}", u2[l][h])] if case["attention"] == "additive" else []
            for key, w in [(f"w{l}_{h}", ws[l][h])] + read:  # vectors the attention does not read are never set
                w = w.detach().numpy()
                err = np.abs(ranks[0][key] - w).max()
                assert err <= 1e-9 * max(np.abs(w).max(), 1.0), (name, key, err)


# ---- the graph transformer -----------------------------------------------------------------------------------------
REACH = ("topA", "nrA", "topB", "nrB", "local_rows", "nA", "nB", "longest")
_GT_REF = {}


def gt_problem(case):
    """(rows, cols, N, cfg, params, X, G, model keywords) of a graph transformer case."""
    M, N, rows, cols = graph(case)
    cfg = W.gt_config(case)
    params, X, G = W.gt_inputs(N, cfg, case["seed"])
    kw = dict(attr=attr_of(rows, cols, cfg["edge_dim"]) if cfg["edge_dim"] else None, beta=cfg["beta"], ffn=cfg["ffn"])
    return rows, cols, N, cfg, params, X, G, kw


def gt_reference(case):
    """The per-entry model's output, dX and parameter gradients, and its output on the rows without entries computed
    from the skip alone (the model on a pattern without entries: M = 0 on every row)."""
    key = (case["gt"], case["mask_seed"])
    if key not in _GT_REF:
        rows, cols, N, cfg, params, X, G, kw = gt_problem(case)
        out, dX, dP = gts.backward_np(rows, cols, N, cfg["layers"], params, X, G, p=cfg["dropout"], seed=case["mask_seed"], **kw)
        none = np.zeros(0, np.int64)
        skip = gts.forward_np(none, none, N, cfg["layers"], params, X, **dict(kw, attr=np.zeros((0, cfg["edge_dim"])) if cfg["edge_dim"] else None))
        _GT_REF[key] = dict(Y=out, dX=dX, dP=dP, skip=skip)
    return _GT_REF[key]


def check_gt_reach(ranks, case, nproc):
    """The case reached what it is for: the configuration's kernel paths (by the tables in the sources), more rows per
    rank than one dw_chunks chunk, at p = 1 a hub row of more than 2000 entries through attention at d >= 64, and at
    p = 4 with c = 1 a rank with entries in one value order only: rank 2 owns the empty third row block, which is its
    A order under local kernel fusion (15d_fusion2: S's own blocks; with edge features, GraphTransformer's branch
    for a rank without A-order attributes) and its B order under replication reuse (15d_fusion1 keeps A-order values
    in the transpose's blocks, which rank 2 holds by S-column)."""
    cfg, tables = W.gt_config(case), kernel_tables()
    att, ln = gt_paths(cfg, tables)
    assert att == tuple(cfg["attention"]) and ln == (tuple(tuple(x) for x in cfg["ln"]) if cfg["ln"] else None), case["name"]
    assert all(int(d["local_rows"]) > tables["min_chunk_rows"] for d in ranks), case["name"]
    if nproc == 1 and max(d for _, d, _ in cfg["layers"]) >= 64:
        assert int(ranks[0]["longest"]) > 2000, case["name"]
    if nproc == 4 and case["c"] == 1:
        empty, full = ("nA", "nB") if case["alg"] == "15d_fusion2" else ("nB", "nA")
        assert int(ranks[2][empty]) == 0 < int(ranks[2][full]), (case["name"], empty)


def check_gt(ranks, case, nproc):
    name = case["name"]
    ranks = ranks_ok(ranks, name)
    check_gt_reach(ranks, case, nproc)
    want = gt_reference(case)
    M, N = W.sizes(case)
    for r, d in enumerate(ranks):
        assert bool(d["repeat"]), (name, r)
    Y = check_rows(ranks, name, "Y", want["Y"], "topA", "nrA")
    check_rows(ranks, name, "dX", want["dX"], "topB", "nrB")
    # the rows without entries take the skip alone: Y = R (beta R with the gate), then the ReLU or the block
    e0, e1 = landmarks(M, N)["empty_rows"]
    assert np.abs(Y[e0:e1] - want["skip"][e0:e1]).max() <= 1e-10 * np.abs(want["Y"]).max(), name
    assert np.abs(want["Y"][e0:e1] - want["skip"][e0:e1]).max() <= 1e-13 * np.abs(want["Y"]).max()
    for l, grads in enumerate(want["dP"]):
        scale = max(np.abs(g).max() for g in grads.values())
        for k, g in grads.items():
            key = f"g{l}_{k}"
            for r, d in enumerate(ranks):
                assert np.array_equal(d[key], ranks[0][key]), (name, r, key, "differs across ranks")
            assert grad_err(ranks[0][key], g, scale) < 1e-10, (name, key, grad_err(ranks[0][key], g, scale))
            assert k == "key_bias" or np.abs(g).max() > 0, (name, key)


def check_gt_steps(ranks, case, want, tparams):
    """Per-step results as tests/test_link_prediction_gpu.check_steps; trained parameters to 1e-9, key_bias within the
    sum of the learning rates (its gradient is rounding noise on both sides, which Adam turns into steps of up to lr);
    everything bit-identical across ranks."""
    name = case["name"]
    for r, d in enumerate(ranks):
        for k in d:
            if k not in REACH and k not in ("scores", "tA_rows", "tA_cols", "H"):
                assert np.array_equal(d[k], ranks[0][k]), (name, r, k, "differs across ranks")
    steps = ranks[0]["steps"]
    assert len(steps) == len(want) == len(case["lrs"])
    for t, w in enumerate(want):
        # From the third step on the gradient norm is as sensitive to rounding as the trained parameters are: the fp64
        # model itself, its entries merely stored in another order, moves the third norm of the "table" case by
        # 1.4e-10 to 2.2e-10 (Adam's first steps have amplified the last bits of the earlier gradients).
        tol = 1e-10 if t < 2 else 1e-9
        assert abs(steps[t][0] - w[0]) <= 1e-10 * abs(w[0]) and abs(steps[t][3] - w[3]) <= tol * abs(w[3]), (name, t, steps[t], w)
        assert (int(steps[t][1]), int(steps[t][2])) == (w[1], w[2]), (name, t, steps[t], w)
    for l, P in enumerate(tparams):
        for k, w in P.items():
            got = ranks[0][f"p{l}_{k}"]
            if k == "key_bias":
                assert np.abs(got - w).max() <= sum(case["lrs"]) * 1.01, (name, l, k)
            else:
                assert np.abs(got - w).max() <= 1e-9 * max(np.abs(w).max(), 1.0), (name, l, k, np.abs(got - w).max())


def check_gt_training(ranks, case, nproc):
    ranks = ranks_ok(ranks, case["name"])
    check_gt_reach(ranks, case, nproc)
    rows, cols, N, cfg, params, X, _, kw = gt_problem(case)
    layers = cfg["layers"]
    labels = W.labels_of(N, layers[-1][1] * layers[-1][2], case["seed"])
    lrs = case["lrs"]
    want, tparams = gts.train_gt(rows, cols, N, layers, params, X, labels, len(lrs), dropout=cfg["dropout"],
                                 seeds=[case["mask_seed"] + 7 * t for t in range(len(lrs))], lr=lrs[0], lrs=lrs,
                                 weight_decay=0.01, max_grad_norm=case.get("clip"), **kw)
    if case.get("clip"):
        assert sum(w[3] > case["clip"] for w in want) == 1, [w[3] for w in want]  # clipping active on one step
    check_gt_steps(ranks, case, want, tparams)


def check_gt_link(ranks, case, nproc):
    name = case["name"]
    ranks = ranks_ok(ranks, name)
    check_gt_reach(ranks, case, nproc)
    rows, cols, N, cfg, params, X, _, kw = gt_problem(case)
    tr, tc, y = W.link_pairs(N, case["seed"])
    lm = landmarks(N, N)
    empty = np.bincount(rows, minlength=N) == 0
    assert np.isin(tr, lm["wide_hubs"]).sum() >= 60 and (empty[tr] & empty[tc]).sum() >= 20 and (tc == lm["hub_col"]).sum() >= 50
    assert (y == 0.25).any() and len(np.unique(tr * N + tc)) < len(tr)
    lrs = case["lrs"]
    want, tparams = gts.link_train_gt(rows, cols, N, cfg["layers"], params, X, (tr, tc, y), len(lrs), dropout=cfg["dropout"],
                                      seeds=[case["mask_seed"] + 7 * t for t in range(len(lrs))], lr=lrs[0], lrs=lrs,
                                      weight_decay=0.01, **kw)
    check_gt_steps(ranks, case, want, tparams)
    # link_evaluate: a forward without dropout; the scores are <H_u, H_v> of the returned buffer in T's A order
    H = assemble(ranks, "H", "topA", "nrA", N)
    wl, wc, wn, _, _, _ = lpo.link_loss(H, H, tr, tc, y, same=True)
    loss, correct, count = ranks[0]["evaluate"]
    assert abs(loss - wl) <= 1e-12 * abs(wl) and int(count) == wn == len(tr) and abs(int(correct) - wc) <= 1, name
    seen = []
    for r, d in enumerate(ranks):
        u, v = d["tA_rows"], d["tA_cols"]
        s = (H[u] * H[v]).sum(1)
        assert np.abs(d["scores"] - s).max(initial=0.0) <= 1e-12 * max(np.abs(s).max(initial=0.0), 1.0), (name, r)
        seen.append(u * N + v)
    assert np.array_equal(np.sort(np.concatenate(seen)), np.sort(tr * N + tc)), name


# ---- PNA, GIN, GINE, GraphSAGE and R-GCN ---------------------------------------------------------------------------
_GNN_REF = {}


def ref_key(case):
    """What a model's reference depends on: the configuration, and the case's aggregation and basis count."""
    cfg = W.gnn_config(case)
    return case["gnn"], cfg.get("aggr"), cfg.get("bases")


def s_relations(case):
    """R-GCN's relation of every entry of graph(case), in its order: hashed on the global tuple list (as the worker's
    ranks take them), then sorted as graph() sorts."""
    M, N = W.sizes(case)
    r, c = (x.astype(np.int64) for x in skewed_tuples(M, N, case["seed"]))
    return W.s_relations(r, c, N)[np.lexsort((c, r))]


def sage_rgcn_model(cfg, rows, cols, rels, N):
    """(params, X) -> the per-entry model's output, for a GraphSAGE or R-GCN configuration."""
    layers, aggr = cfg["layers"], cfg["aggr"]
    if cfg["model"] == "sage":
        return lambda tp, x: gsa.model_torch(rows, cols, N, layers, tp, x, aggr)
    if cfg.get("bases"):
        return lambda tp, x: bo.model_torch(rows, cols, rels, N, layers, tp, x, W.NUM_RELATIONS, cfg["bases"], aggr)
    return lambda tp, x: ro.model_torch(rows, cols, rels, N, layers, tp, x, W.NUM_RELATIONS, aggr)



def gnn_problem(case):
    """(rows, cols, N, cfg, params, X, G, oracle) of a PNA / GIN / GraphSAGE / R-GCN case; oracle: PNA's (aggregators,
    scalers, avg_lin, avg_log) from the graph's own degree histogram, GINE's per-entry attributes (None for GIN), or
    R-GCN's relations (None for GraphSAGE)."""
    M, N, rows, cols = graph(case)
    cfg = W.gnn_config(case)
    params, X, G = W.gnn_inputs(N, cfg, case["seed"])
    if cfg["model"] == "pna":
        hist = np.bincount(np.bincount(rows, minlength=N))
        oracle = (cfg["aggregators"], cfg["scalers"], *po.degree_averages(hist))
    elif cfg["model"] == "rgcn":
        oracle = s_relations(case)
    elif cfg["model"] == "sage":
        oracle = None
    else:
        oracle = go.attr_of(rows, cols, cfg["edge_dim"]) if cfg["edge_dim"] else None
    return rows, cols, N, cfg, params, X, G, oracle


def gnn_reference(case):
    """The per-entry model's output, dX and parameter gradients, and its output on a pattern without entries (what the
    rows without entries must give: PNA's post([x, 0..]) with d clamped to 1, GIN's MLP of (1 + eps) x)."""
    key = ref_key(case)
    if key not in _GNN_REF:
        rows, cols, N, cfg, params, X, G, oracle = gnn_problem(case)
        layers = cfg["layers"]
        none = np.zeros(0, np.int64)
        tp = [{k: po._t(v) for k, v in P.items()} for P in params]
        if cfg["model"] == "sage":
            Y, dX, dP = gsa.forward_backward(rows, cols, N, layers, params, X, cfg["aggr"], G)
            alone = sage_rgcn_model(cfg, none, none, np.zeros(0), N)(tp, po._t(X))
        elif cfg["model"] == "rgcn" and cfg.get("bases"):
            Y, dX, dP = bo.forward_backward(rows, cols, oracle, N, layers, params, X, W.NUM_RELATIONS, cfg["bases"], cfg["aggr"], G)
            alone = sage_rgcn_model(cfg, none, none, np.zeros(0), N)(tp, po._t(X))
        elif cfg["model"] == "rgcn":
            Y, dX, dP = ro.forward_backward(rows, cols, oracle, N, layers, params, X, W.NUM_RELATIONS, cfg["aggr"], G)
            alone = sage_rgcn_model(cfg, none, none, np.zeros(0), N)(tp, po._t(X))
        elif cfg["model"] == "pna":
            Y, dX, dP = po.forward_backward(rows, cols, N, layers, params, X, G, *oracle)
            alone = po.model_torch(none, none, N, layers, tp, po._t(X), *oracle)
        else:
            Y, dX, dP = go.forward_backward(rows, cols, N, layers, params, X, G, oracle)
            attr = None if oracle is None else torch.zeros(0, cfg["edge_dim"], dtype=torch.float64)
            alone = go.model_torch(none, none, N, layers, tp, go._t(X), attr)
        _GNN_REF[key] = dict(Y=Y, dX=dX, dP=dP, alone=alone.detach().numpy())
    return _GNN_REF[key]


def check_gnn_reach(ranks, case, nproc):
    """More rows per rank than one reduction chunk, at p = 1 a hub row of more than 2000 entries, and at p = 4 with
    c = 1 a rank without entries in one value order (rank 2's row block is the empty third one; see check_gt_reach):
    under 15d_fusion2 that is the A order, so GINE's edge projection and its dW_e run on 0 rows there."""
    tables = kernel_tables()
    assert all(int(d["local_rows"]) > tables["min_chunk_rows"] for d in ranks), case["name"]
    if nproc == 1:
        assert int(ranks[0]["longest"]) > 2000, case["name"]
    if nproc == 4 and case["c"] == 1:
        empty, full = ("nA", "nB") if case["alg"] == "15d_fusion2" else ("nB", "nA")
        assert int(ranks[2][empty]) == 0 < int(ranks[2][full]), (case["name"], [int(d["nA"]) for d in ranks])


def check_gnn(ranks, case, nproc):
    name = case["name"]
    ranks = ranks_ok(ranks, name)
    check_gnn_reach(ranks, case, nproc)
    want = gnn_reference(case)
    M, N, rows, _ = graph(case)
    cfg = W.gnn_config(case)
    for r, d in enumerate(ranks):
        assert bool(d["repeat"]), (name, r)
    Y = check_rows(ranks, name, "Y", want["Y"], "topA", "nrA")
    check_rows(ranks, name, "dX", want["dX"], "topB", "nrB")
    # the rows without entries (the empty third row block, every row % 9 == 4) take their own input alone
    empty = np.bincount(rows, minlength=M) == 0
    e0, e1 = landmarks(M, N)["empty_rows"]
    assert empty[e0:e1].all() and empty[list(W.TIE_ROWS)].all()
    scale = np.abs(want["Y"]).max()
    assert np.abs(Y[empty] - want["alone"][empty]).max() <= 1e-10 * scale, name
    assert np.abs(want["Y"][empty] - want["alone"][empty]).max() <= 1e-13 * scale
    train_eps = case.get("train_eps", True)
    for l, grads in enumerate(want["dP"]):
        gscale = max(np.abs(g).max() for g in grads.values())
        for k, g in grads.items():
            key = f"g{l}_{k}"
            for r, d in enumerate(ranks):
                assert np.array_equal(d[key], ranks[0][key]), (name, r, key, "differs across ranks")
            if k == "eps" and not train_eps:  # a constant: its gradient reads 0
                assert not ranks[0][key].any(), (name, key)
                continue
            assert np.abs(g).max() > 0, (name, key)
            assert grad_err(ranks[0][key], g, gscale) < 1e-10, (name, key, grad_err(ranks[0][key], g, gscale))
    if cfg["model"] in ("sage", "rgcn"):  # rows without entries and with equal inputs, on ranks 0 and 3 at p = 4
        assert np.array_equal(Y[W.TIE_ROWS[0]], Y[W.TIE_ROWS[1]]), name
    if cfg["model"] == "rgcn":  # the relation no entry carries: its weight block (its row of comp) gets exactly 0
        U = W.USED_RELATIONS
        for l, (f, _) in enumerate(cfg["layers"]):
            g = ranks[0][f"g{l}_comp"][U:] if cfg.get("bases") else ranks[0][f"g{l}_weight"][U * f:]
            assert g.size and not g.any(), (name, l, "the unused relation has a gradient")
    if cfg["model"] == "gin" and cfg["edge_dim"] and nproc == 4 and case["alg"] == "15d_fusion2" and case["c"] == 1:
        # a rank without A-order entries adds nothing to dW_e; the all-reduced dW_e above matched the model
        assert [int(d["nA"]) for d in ranks].count(0) >= 1, name


def check_gine_int(ranks, case, nproc):
    """edge_relu_aggregate on integers: A, dX and dE equal numpy exactly, on every rank; the copies of a duplicate get
    bit-equal dE; X_v + E_i == 0 happens on the hub row (the strict mask decides those entries); rows without entries
    give A = 0 and the untouched columns dX = 0."""
    name = case["name"]
    ranks = ranks_ok(ranks, name)
    M, N, rows, cols = graph(case)
    f = case["R"]
    X, dA = W.gine_int_inputs(N, f, case["seed"])
    E = go.edge_rows(rows, cols, f)
    lm = landmarks(M, N)
    hub = rows == lm["wide_hubs"][0]
    assert ((X[cols] + E == 0) & hub[:, None]).sum() > 100
    A = go.edge_relu_aggregate(rows, cols, M, X, E)
    dX, dE = go.edge_relu_aggregate_backward(rows, cols, X, E, dA, N)
    assert np.abs(A).max() < 2 ** 20 and np.abs(dX).max() < 2 ** 20  # integers: every partial sum is exact
    for r, d in enumerate(ranks):
        assert bool(d["repeat"]), (name, r)
        for key, want, top, nr in (("A", A, "topA", "nrA"), ("dX", dX, "topB", "nrB")):
            t, n = int(d[top]), min(int(d[nr]), len(want) - int(d[top]))
            assert np.array_equal(d[key][:n], want[t:t + n]), (name, r, key)
        assert np.array_equal(d["dE"], lookup(N, rows, cols, dE, d["rA"], d["cA"])), (name, r, "dE")
    Ag, dXg = assemble(ranks, "A", "topA", "nrA", M), assemble(ranks, "dX", "topB", "nrB", N)
    assert not Ag[np.bincount(rows, minlength=M) == 0].any() and not dXg[lm["empty_cols"][0]:lm["empty_cols"][1]].any()
    keys = np.concatenate([d["rA"] * N + d["cA"] for d in ranks])
    vals = np.concatenate([d["dE"] for d in ranks])
    order = np.argsort(keys, kind="stable")
    keys, vals = keys[order], vals[order]
    same = np.flatnonzero(np.diff(keys) == 0)
    assert len(same) >= 50 and np.array_equal(vals[same], vals[same + 1]), (name, "copies of a duplicate differ")


_GNN_TRAIN_REF = {}


def gnn_train_reference(case):
    """(per-step results, trained parameters, trained head or None) of the per-entry model."""
    key = (ref_key(case), case["task"], case.get("pool"), case.get("train_eps", True))
    if key in _GNN_TRAIN_REF:
        return _GNN_TRAIN_REF[key]
    rows, cols, N, cfg, params, X, _, oracle = gnn_problem(case)
    layers, steps = cfg["layers"], case["steps"]
    pna, train_eps = cfg["model"] == "pna", case.get("train_eps", True)
    head = None
    if cfg["model"] in ("sage", "rgcn"):
        model = sage_rgcn_model(cfg, rows, cols, oracle, N)
        tp, x = gsa._leaves(params), gsa._t(X)
        fwd = lambda _: model(tp, x)  # noqa: E731
        leaves = [v for P in tp for v in P.values()]
        if case["task"] == "node":
            res = tro.train(fwd, leaves, W.labels_of(N, layers[-1][-1], case["seed"]), steps, lr=W.GNN_LR)
        elif case["task"] == "link":
            res = lpo.link_train_step(W.link_pairs(N, case["seed"]))(fwd, leaves, None, steps, lr=W.GNN_LR)
        else:
            batch, G, labels = W.readout_batch(N, case["seed"])
            res, head = gro.train(fwd, leaves, batch, G, case["pool"], W.readout_head(layers[-1][-1], case["seed"]), labels, steps,
                                  lr=W.GNN_LR)
        trained = [{k: v.detach().numpy().copy() for k, v in P.items()} for P in tp]
    elif case["task"] == "node":
        labels = W.labels_of(N, layers[-1][-1], case["seed"])
        if pna:
            res, trained = po.train(rows, cols, N, layers, params, X, oracle, labels, steps, lr=W.GNN_LR)
        else:
            res, trained = go.train(rows, cols, N, layers, params, X, labels, steps, attr=oracle, train_eps=train_eps, lr=W.GNN_LR)
    elif case["task"] == "link":
        pairs = W.link_pairs(N, case["seed"])
        if pna:
            res, trained = po.train_link(rows, cols, N, layers, params, X, oracle, pairs, steps, lr=W.GNN_LR)
        else:
            res, trained = go.train_link(rows, cols, N, layers, params, X, pairs, steps, attr=oracle, train_eps=train_eps, lr=W.GNN_LR)
    else:
        batch, G, labels = W.readout_batch(N, case["seed"])
        tp = po._leaves(params) if pna else go._leaves(params, train_eps)
        x = po._t(X)
        if pna:
            fwd = lambda _: po.model_torch(rows, cols, N, layers, tp, x, *oracle)  # noqa: E731
            leaves = [v for P in tp for v in P.values()]
        else:
            attr = None if oracle is None else go._t(oracle)
            fwd = lambda _: go.model_torch(rows, cols, N, layers, tp, x, attr)  # noqa: E731
            leaves = go._trained(tp)
        res, head = gro.train(fwd, leaves, batch, G, case["pool"], W.readout_head(layers[-1][-1], case["seed"]), labels, steps, lr=W.GNN_LR)
        trained = [{k: v.detach().numpy().copy() for k, v in P.items()} for P in tp]
    _GNN_TRAIN_REF[key] = (res, trained, head)
    return _GNN_TRAIN_REF[key]


def check_gnn_training(ranks, case, nproc):
    """Three steps against the per-entry model with torch's AdamW: losses to 1e-10; gradient norms and trained
    parameters to 1e-9, since Adam's g / (sqrt(v) + eps) amplifies the last bits of the earlier gradients (the graph
    transformer's cases measured the fp64 model itself, its entries merely reordered, moving the third norm by 2.2e-10);
    correct and labelled exactly; everything bit-identical across ranks."""
    name = case["name"]
    ranks = ranks_ok(ranks, name)
    check_gnn_reach(ranks, case, nproc)
    for r, d in enumerate(ranks):
        for k in d:
            if k not in REACH:
                assert np.array_equal(d[k], ranks[0][k]), (name, r, k, "differs across ranks")
    # the graph cases' batch (a graph over every row block with a hub row, a maximum on two ranks, an empty graph) is
    # checked by tests/test_skewed_gnn_fixture.py
    want, trained, head = gnn_train_reference(case)
    steps = ranks[0]["steps"]
    assert len(steps) == len(want) == case["steps"]
    for t, w in enumerate(want):
        assert abs(steps[t][0] - w[0]) <= 1e-10 * abs(w[0]) and abs(steps[t][3] - w[3]) <= 1e-9 * abs(w[3]), (name, t, steps[t], w)
        assert (int(steps[t][1]), int(steps[t][2])) == (w[1], w[2]), (name, t, steps[t], w)
    for l, P in enumerate(trained):
        for k, w in P.items():
            got = ranks[0][f"p{l}_{k}"]
            assert np.abs(got - w).max() <= 1e-9 * max(np.abs(w).max(), 1.0), (name, l, k, np.abs(got - w).max())
    if head is not None:
        for k, w in zip(("weight", "bias"), head):
            assert np.abs(ranks[0][f"head_{k}"] - w).max() <= 1e-9 * max(np.abs(w).max(), 1.0), (name, k)


# ---- max aggregation, DistMult and relational link training ------------------------------------------------------
def check_max_agg(ranks, case, nproc):
    """Z and C equal the model exactly on every rank (C counts both copies of a duplicate, and the exact zeros of X
    tie), dX to 1e-12; a hub row of more than 2000 entries at p = 1, a rank without A-order entries at p = 4 on
    15d_fusion2."""
    name = case["name"]
    ranks = ranks_ok(ranks, name)
    M, N, rows, cols = graph(case)
    X, dZ = W.max_agg_inputs(N, case["R"], case["seed"])
    Z, C = gsa.max_aggregate(rows, cols, M, X)
    dX = gsa.max_aggregate_backward(rows, cols, Z, C, dZ, N, X)
    # both copies of a duplicate attain a positive maximum somewhere, and ties (mostly at 0) fill 4 % of the cells
    dup = np.flatnonzero(np.diff(rows * N + cols) == 0)
    has = np.bincount(rows, minlength=M) > 0
    assert ((X[cols[dup]] == Z[rows[dup]]) & (Z[rows[dup]] > 0)).any() and (C[has] >= 2).mean() > 0.04
    for r, d in enumerate(ranks):
        assert bool(d["repeat"]), (name, r)
        t, n = int(d["topA"]), min(int(d["nrA"]), M - int(d["topA"]))
        for key, want in (("Z", Z), ("C", C)):
            assert np.array_equal(d[key][:n], want[t:t + n]), (name, r, key)
    check_rows(ranks, name, "dX", dX, "topB", "nrB", tol=1e-12)
    if nproc == 1:
        assert int(ranks[0]["longest"]) > 2000, name
    if nproc == 4 and case["alg"] == "15d_fusion2" and case["c"] == 1:
        assert int(ranks[2]["nA"]) == 0 < int(ranks[3]["nA"]), name


_DM_REF = {}


def distmult_reference(case):
    """(T_pos, T_neg, the positive call's and the negative call's dmo.op results) of a distmult case."""
    key = (W.sizes(case), case["R"])
    if key not in _DM_REF:
        N = W.sizes(case)[1]
        pos, neg = W.distmult_targets(N, case["seed"])
        H, rel = W.distmult_inputs(N, case["R"], case["seed"])
        inv = 1.0 / (len(pos[0]) + len(neg[0]))
        _DM_REF[key] = (pos, neg, dmo.op(H, H, rel, *pos, 1.0, inv, same=True), dmo.op(H, H, rel, *neg, 0.0, inv, same=True))
    return _DM_REF[key]


def check_distmult_reach(ranks, case, nproc, pos, N):
    """Relation 0 spans more than one HNH_EDGE_PIECE on every rank with T entries (more than 8, one per warp of the
    dD sum, at p = 1); at p = 1 a hub row of more than 2000 pairs; at p = 4 on 15d_fusion2 rank 2 holds no T entry."""
    keys0 = (pos[0] * N + pos[1])[pos[2] == 0]
    for r, d in enumerate(ranks):
        if len(d["erp"]):
            n0 = np.isin(keys0, d["erp"] * N + d["ecp"]).sum()
            assert n0 > PIECE * (8 if nproc == 1 else 1), (case["name"], r, n0)
    if nproc == 1:
        assert np.bincount(ranks[0]["erp"]).max() > 2000, case["name"]
    if nproc == 4 and case["alg"] == "15d_fusion2" and case["c"] == 1:
        assert [len(d["erp"]) for d in ranks].count(0) == 1, (case["name"], [len(d["erp"]) for d in ranks])


def check_distmult(ranks, case, nproc):
    """A positive call and an accumulated negative one against dmo.op: the (loss, correct) sums and dD bit-identical on
    every rank, correct exactly (no score lies near 0), the loss, dD and dH to 1e-12, every pair's scores as a multiset,
    and dD's row of the relation no pair carries exactly 0."""
    name = case["name"]
    ranks = ranks_ok(ranks, name)
    N = W.sizes(case)[1]
    pos, neg, (lp, cp, sp, gp, _, dp), (ln, cn, sn, gn, _, dn) = distmult_reference(case)
    U = W.USED_RELATIONS
    assert (pos[2] < U).all() and (neg[2] < U).all() and not (dp + dn)[U:].any()
    check_distmult_reach(ranks, case, nproc, pos, N)
    for r, d in enumerate(ranks):
        assert bool(d["repeat"]), (name, r)
        assert np.array_equal(d["res"], ranks[0]["res"]) and np.array_equal(d["dD"], ranks[0]["dD"]), (name, r, "differs across ranks")
        assert not d["dD"][U:].any(), (name, r, "the relation no pair carries has a gradient")
        assert _scores_match(d["sp"], d["erp"], d["ecp"], pos, sp) and _scores_match(d["sn"], d["ern"], d["ecn"], neg, sn), (name, r)
    for er, ec, trip in (("erp", "ecp", pos), ("ern", "ecn", neg)):  # every copy of every pair on some rank
        seen = np.concatenate([d[er] * N + d[ec] for d in ranks])
        assert np.array_equal(np.sort(seen), np.sort(trip[0] * N + trip[1])), (name, er)
    res = ranks[0]["res"]
    assert abs(res[0][0] - lp) <= 1e-12 * lp and abs(res[1][0] - ln) <= 1e-12 * ln, (name, res, lp, ln)
    assert (int(res[0][1]), int(res[1][1])) == (cp, cn), (name, res, cp, cn)
    assert rel_err(ranks[0]["dD"], dp + dn) < 1e-12, name
    check_rows(ranks, name, "dH", gp + gn, "topA", "nrA", tol=1e-12)


def check_rel_link(ranks, case, nproc):
    """Relational link train steps against dmo.train over the per-entry model, as check_gnn_training (and rel to 1e-9),
    the unused relation's row of drel exactly 0, then relational_link_evaluate against dmo.relational_loss on the
    returned H and rel."""
    name = case["name"]
    ranks = ranks_ok(ranks, name)
    check_gnn_reach(ranks, case, nproc)
    for r, d in enumerate(ranks):
        for k in d:
            if k not in REACH and k not in ("sp", "sn", "erp", "ecp", "ern", "ecn", "H"):
                assert np.array_equal(d[k], ranks[0][k]), (name, r, k, "differs across ranks")
    rows, cols, N, cfg, params, X, _, rels = gnn_problem(case)
    pos, neg = W.distmult_targets(N, case["seed"])
    model = sage_rgcn_model(cfg, rows, cols, rels, N)
    tp, x = gsa._leaves(params), gsa._t(X)
    rel0 = W.distmult_inputs(N, cfg["layers"][-1][-1], case["seed"])[1]
    want, rel = dmo.train(lambda _: model(tp, x), [v for P in tp for v in P.values()], rel0, pos, neg, case["steps"], lr=W.GNN_LR)
    steps = ranks[0]["steps"]
    assert len(steps) == len(want) == case["steps"]
    for t, w in enumerate(want):
        assert abs(steps[t][0] - w[0]) <= 1e-10 * abs(w[0]) and abs(steps[t][3] - w[3]) <= 1e-9 * abs(w[3]), (name, t, steps[t], w)
        assert (int(steps[t][1]), int(steps[t][2])) == (w[1], w[2]), (name, t, steps[t], w)
    trained = {f"p{l}_{k}": v.detach().numpy() for l, P in enumerate(tp) for k, v in P.items()}
    for k, w in dict(trained, rel=rel).items():
        assert np.abs(ranks[0][k] - w).max() <= 1e-9 * max(np.abs(w).max(), 1.0), (name, k, np.abs(ranks[0][k] - w).max())
    assert not ranks[0]["drel"][W.USED_RELATIONS:].any() and ranks[0]["drel"].any(), name
    H = assemble(ranks, "H", "topA", "nrA", N)
    loss, correct, count, sp, sn = dmo.relational_loss(dmo._t(H), dmo._t(ranks[0]["rel"]), pos, neg)
    got = ranks[0]["evaluate"]
    assert abs(got[0] - float(loss)) <= 1e-12 * abs(float(loss)) and (int(got[1]), int(got[2])) == (correct, count), (name, got)
    for r, d in enumerate(ranks):
        assert _scores_match(d["sp"], d["erp"], d["ecp"], pos, sp) and _scores_match(d["sn"], d["ern"], d["ecn"], neg, sn), (name, r)


# ---- across rank counts --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nproc", [2, 4])
def test_results_do_not_depend_on_the_rank_count(nproc):
    """Every attention, GAT, graph transformer, PNA / GIN and training case that also runs at p = 1: the assembled global
    result equals p = 1's to 1e-12 of its largest entry (the sums run in another order), +-inf exactly; trained
    parameters to 1e-9; the integer GINE aggregation bit for bit."""
    one, many = results(1), results(nproc)
    checked = 0
    for case in CASES[nproc]:
        name = case["name"]
        if name not in one or case["kind"] not in ("attn", "gat", "train", "gt", "gt_train", "gt_link", "gnn", "gnn_train",
                                                   "gine_int", "max_agg", "distmult", "rel_link") or case.get("rejected"):
            continue
        a, b = ranks_ok(one[name], name), ranks_ok(many[name], name)
        M, N = W.sizes(case)
        if case["kind"] == "max_agg":  # Z and C are exact on any layout
            for key in ("Z", "C"):
                assert np.array_equal(assemble(b, key, "topA", "nrA", M), assemble(a, key, "topA", "nrA", M)), (name, nproc, key)
            assert rel_err(assemble(b, "dX", "topB", "nrB", N), assemble(a, "dX", "topB", "nrB", N)) < 1e-12, (name, nproc)
            checked += 1
            continue
        if case["kind"] == "distmult":
            ra, rb = a[0]["res"], b[0]["res"]
            assert np.array_equal(ra[:, 1], rb[:, 1]) and rel_err(rb[:, 0], ra[:, 0]) < 1e-12, (name, nproc)
            assert rel_err(b[0]["dD"], a[0]["dD"]) < 1e-12, (name, nproc)
            assert rel_err(assemble(b, "dH", "topA", "nrA", M), assemble(a, "dH", "topA", "nrA", M)) < 1e-12, (name, nproc)
            checked += 1
            continue
        if case["kind"] == "rel_link":
            for k in a[0]:
                if k in ("steps", "rel") or k.startswith("p"):
                    assert rel_err(b[0][k], a[0][k]) < 1e-9, (name, nproc, k)
            checked += 1
            continue
        if case["kind"] == "gine_int":  # integers: the same on any layout, bit for bit
            for key, top, nr, total in (("A", "topA", "nrA", M), ("dX", "topB", "nrB", N)):
                assert np.array_equal(assemble(b, key, top, nr, total), assemble(a, key, top, nr, total)), (name, nproc, key)
            checked += 1
            continue
        if case["kind"] in ("gt", "gnn"):
            for key in ("Y", "dX"):
                top, nr, total = ("topA", "nrA", M) if key == "Y" else ("topB", "nrB", N)
                assert rel_err(assemble(b, key, top, nr, total), assemble(a, key, top, nr, total)) < 1e-12, (name, nproc, key)
            cfg = W.gt_config(case) if case["kind"] == "gt" else W.gnn_config(case)
            for l in range(len(cfg["layers"])):
                grads = {k: v for k, v in a[0].items() if k.startswith(f"g{l}_")}
                scale = max(np.abs(g).max() for g in grads.values())  # key_bias, a constant eps: 0 (up to rounding)
                for k, g in grads.items():
                    assert grad_err(b[0][k], g, scale) < 1e-12, (name, nproc, k)
            checked += 1
            continue
        if case["kind"] == "gnn_train":
            for k in a[0]:
                if k == "steps" or k.startswith("p") or k.startswith("head_"):
                    assert rel_err(b[0][k], a[0][k]) < 1e-9, (name, nproc, k)
            checked += 1
            continue
        if case["kind"] in ("gt_train", "gt_link"):
            for k in a[0]:
                if k.endswith("key_bias"):  # Adam's steps of up to lr on a rounding-noise gradient
                    assert np.abs(b[0][k] - a[0][k]).max() <= sum(case["lrs"]) * 1.01, (name, nproc, k)
                elif k == "steps" or k.startswith("p"):
                    assert rel_err(b[0][k], a[0][k]) < 1e-9, (name, nproc, k)
            checked += 1
            continue
        if case["kind"] == "train":
            pairs = [(a[0][k], b[0][k]) for k in a[0] if k != "local_rows"]
        else:
            keysA, keysB = (("Z", "L", "dQ"), ("dK", "dV")) if case["kind"] == "attn" else (("out",), ("dX0",))
            pairs = [(assemble(a, k, "topA", "nrA", M), assemble(b, k, "topA", "nrA", M)) for k in keysA]
            pairs += [(assemble(a, k, "topB", "nrB", N), assemble(b, k, "topB", "nrB", N)) for k in keysB]
        for x, y in pairs:
            # trained parameters: AdamW's g / (sqrt(v) + eps) amplifies the last bits of small gradients, as against the model
            assert rel_err(y, x) < (1e-9 if case["kind"] == "train" else 1e-12), (name, nproc)
        checked += 1
    assert checked >= 10


@pytest.mark.parametrize("nproc", [2, 4])
def test_layouts_without_the_op_still_refuse_on_every_rank(nproc):
    got = results(nproc)
    rejected = [c for c in CASES[nproc] if c.get("rejected")]
    assert rejected
    for c in rejected:
        for r, d in enumerate(got[c["name"]]):
            msg = str(d.get("error"))
            assert "error" in d and "code -1" in msg and "not defined for" in msg and f"p = {nproc}" in msg, (c["name"], r, msg)


@pytest.mark.parametrize("nproc,case", params("base"))
def test_base_ops_on_the_skewed_graph(nproc, case):
    check_base(results(nproc)[case["name"]], case, nproc)


@pytest.mark.parametrize("nproc,case", params("softmax"))
def test_edge_softmax_on_the_skewed_graph(nproc, case):
    check_softmax(results(nproc)[case["name"]], case, nproc)


@pytest.mark.parametrize("nproc,case", params("attn"))
def test_sparse_attention_on_the_skewed_graph(nproc, case):
    check_attention(results(nproc)[case["name"]], case, nproc)


@pytest.mark.parametrize("nproc,case", params("gat"))
def test_gat_on_the_skewed_graph(nproc, case):
    check_gat(results(nproc)[case["name"]], case, nproc)


@pytest.mark.parametrize("nproc,case", params("train"))
def test_gat_training_on_the_skewed_graph(nproc, case):
    check_training(results(nproc)[case["name"]], case, nproc)


@pytest.mark.parametrize("nproc,case", params("gt"))
def test_graph_transformer_on_the_skewed_graph(nproc, case):
    check_gt(results(nproc)[case["name"]], case, nproc)


@pytest.mark.parametrize("nproc,case", params("gt_train"))
def test_graph_transformer_training_on_the_skewed_graph(nproc, case):
    check_gt_training(results(nproc)[case["name"]], case, nproc)


@pytest.mark.parametrize("nproc,case", params("gt_link"))
def test_graph_transformer_link_training_on_the_skewed_graph(nproc, case):
    check_gt_link(results(nproc)[case["name"]], case, nproc)


@pytest.mark.parametrize("nproc,case", params("gnn"))
def test_pna_and_gin_on_the_skewed_graph(nproc, case):
    check_gnn(results(nproc)[case["name"]], case, nproc)


@pytest.mark.parametrize("nproc,case", params("gine_int"))
def test_gine_aggregation_on_integers_on_the_skewed_graph(nproc, case):
    check_gine_int(results(nproc)[case["name"]], case, nproc)


@pytest.mark.parametrize("nproc,case", params("gnn_train"))
def test_pna_and_gin_training_on_the_skewed_graph(nproc, case):
    check_gnn_training(results(nproc)[case["name"]], case, nproc)


@pytest.mark.parametrize("nproc,case", params("max_agg"))
def test_max_aggregation_on_the_skewed_graph(nproc, case):
    check_max_agg(results(nproc)[case["name"]], case, nproc)


@pytest.mark.parametrize("nproc,case", params("distmult"))
def test_distmult_loss_on_the_skewed_graph(nproc, case):
    check_distmult(results(nproc)[case["name"]], case, nproc)


@pytest.mark.parametrize("nproc,case", params("rel_link"))
def test_relational_link_training_on_the_skewed_graph(nproc, case):
    check_rel_link(results(nproc)[case["name"]], case, nproc)
