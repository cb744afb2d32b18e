"""The skewed graph of tests/skewed_graph.py on one rank, in-process: the op table of
tests/test_skewed_graphs_multirank_gpu.py (its cases, worker code and checks) on all five algorithms and on the
rectangular variants, every graph transformer configuration (and its refusal of the rectangular sizes), every PNA / GIN
configuration and GINE's integer edge-ReLU aggregation on all five algorithms, every GraphSAGE and R-GCN configuration
and max_aggregate and distmult_loss at every width of the multi-rank cases on all five algorithms, and the
kernel-level entry points fed one skewed block directly -- the sparse-attention step, finish, grad_q and grad_kv kernels
on the block and on its transpose (where the hub column is one very long row), and the edge-softmax plan, statistics,
apply and backward kernels keyed by row and by column -- so that a failure on several ranks can be told apart from a
kernel fault."""
import numpy as np
import pytest

from distributed_sddmm_b200 import driver as D
from tests import gat_softmax_oracle as gso
from tests import mp_skewed_worker as W
from tests import test_skewed_graphs_multirank_gpu as T
from tests.skewed_graph import RECTANGULAR, landmarks, skewed_tuples
from tests.test_edge_softmax_gpu import _backward, _plan, _softmax
from tests.test_sparse_attention_gpu import _check_kernels, _csr

pytestmark = pytest.mark.gpu
ALGS = ["15d_fusion1", "15d_fusion2", "15d_sparse", "25d_dense_replicate", "25d_sparse_replicate"]


@pytest.fixture(scope="module")
def world():
    D.world_init("self")
    yield
    D.world_finalize()


def _attn(alg, heads, d, variant, dropout=0.0, **kw):
    return dict(T._case("attn", alg, 1, heads * d, heads=heads, d=d, variant=variant, dropout=dropout, mask_seed=29), **kw)


def _cases(alg, i):
    """One width per algorithm from each op's list, rotated so that the five algorithms cover all of them."""
    shapes = [(2, 64), (1, 128), (4, 7)]
    variants = [("plain", 0.0), ("plain", 0.4), ("bias", 0.4), ("edge", 0.0), ("edge", 0.4)]
    out = [T._case("base", alg, 1, [64, 128, 256, 100][i % 4], script=T.ALL_OPS),
           T._case("softmax", alg, 1, 8, mask=i % 2)]
    out += [_attn(alg, *shapes[(i + j) % 3], *variants[(i + j) % 5]) for j in range(3)]
    out.append(T._case("gat", alg, 1, 64, attention=["leaky", "softmax", "additive", "gatv2"][i % 4], layers=T.GAT_LAYERS))
    return out


CHECKS = dict(base=T.check_base, softmax=T.check_softmax, attn=T.check_attention, gat=T.check_gat, train=T.check_training,
              gt=T.check_gt, gnn=T.check_gnn, gine_int=T.check_gine_int, max_agg=T.check_max_agg, distmult=T.check_distmult)
P1 = [c for i, alg in enumerate(ALGS) for c in _cases(alg, i)]
P1 += [T._case("train", "25d_dense_replicate", 1, 64, attention="additive", layers=T.GAT_LAYERS, steps=3)]
# the graph transformer: every configuration on 15d_fusion1, the two with edge features on every algorithm
P1 += [T.gt_case("gt", alg, 1, name) for name in ("table", "odd") for alg in ALGS]
P1 += [T.gt_case("gt", "15d_fusion1", 1, name) for name in ("wide_heads", "ln_backward_generic", "ln_generic")]
# PNA, GIN and GINE: every configuration and the integer op on every algorithm
P1 += [T.gnn_case("gnn", alg, 1, name) for name in W.GNN_CONFIGS for alg in ALGS]
P1 += [T._case("gine_int", alg, 1, W.GINE_INT_WIDTH) for alg in ALGS]
# GraphSAGE and R-GCN: every configuration and aggregation; max_aggregate and distmult_loss at every width; on every algorithm
P1 += [T.gnn_case("gnn", alg, 1, name, **kw) for name, kw in T.SAGE_RGCN_TABLE + T.SAGE_RGCN_OTHER for alg in ALGS]
P1 += [T._case(kind, alg, 1, f) for kind, widths in (("max_agg", W.MAX_AGG_WIDTHS), ("distmult", W.DISTMULT_WIDTHS))
       for f in widths for alg in ALGS]
RECT = [dict(c, m=M, n=N) for k, (M, N) in enumerate(RECTANGULAR)
        for c in (T._case("base", ALGS[k], 1, 128, script=T.ALL_OPS), T._case("softmax", ALGS[k + 2], 1, 8, mask=1),
                  _attn(ALGS[k + 3], 2, 64, "bias", 0.4), _attn(ALGS[k], 1, 128, "edge"))]


@pytest.mark.parametrize("case", P1 + RECT, ids=lambda c: c["name"] + (f"_{c['m']}x{c['n']}" if "m" in c else ""))
def test_p1_ops_on_the_skewed_graph(world, case):
    CHECKS[case["kind"]]([W.run_case(D, case, 0, 1)], case, 1)


@pytest.mark.parametrize("M,N", RECTANGULAR)
def test_graph_transformer_refuses_rectangular_sizes(world, M, N):
    """A and B layouts of other row counts: the constructor raises, before any launch."""
    out = W.run_case(D, dict(T.gt_case("gt", "15d_fusion1", 1, "odd"), m=M, n=N, rejected=1), 0, 1)
    msg = str(out.get("error"))
    assert "code -1" in msg and "GraphTransformer" in msg, msg


def _block(M, N, seed=5):
    r, c = (x.astype(np.int64) for x in skewed_tuples(M, N, seed))
    order = np.lexsort((c, r))
    return r[order], c[order]


@pytest.mark.parametrize("d", [64, 128, 7])
@pytest.mark.parametrize("M,N", [(4200, 4200), RECTANGULAR[0]])
def test_attention_kernels_on_a_skewed_block_and_its_transpose(world, M, N, d):
    """_check_kernels runs step + finish and grad_q on the block and grad_kv on its transpose, against the fp64 model,
    twice for the bits: the transpose's row of the hub column holds more than 60 % of the rows with entries."""
    rr, cc = _block(M, N)
    rowStart, rr, cc = _csr(rr, cc, M)
    assert np.bincount(cc).max() > 0.6 * (np.diff(rowStart) > 0).sum() and np.diff(rowStart).max() > 2100
    _check_kernels(rowStart, rr, cc, M, N, d, np.random.default_rng(T.SEED + d), False, 0, 0)


@pytest.mark.parametrize("by", ["row", "column"])
def test_edge_softmax_kernels_on_a_skewed_block(world, by):
    """Plan, statistics, apply, dot and backward keyed by the block's rows (hub rows of three pieces) and by its columns
    (the transpose: one hub row, most others short), entries in the shuffled order the generator returns."""
    import torch
    from distributed_sddmm_b200 import lib
    L, dev = lib(), torch.device("cuda:0")
    M = N = 4200
    r, c = (x.astype(np.int64) for x in skewed_tuples(M, N, 5))
    keys, n = (r, M) if by == "row" else (c, N)
    pl = _plan(L, torch, dev, keys, n)
    lens = np.bincount(keys, minlength=n)
    assert pl["P"] == int(np.sum((lens + 1023) // 1024)) and lens.max() > (2048 if by == "row" else 1024)
    x_np = W.score(r, c)
    x_np[W.masked(r, c, M, N) & (lens[keys] > 40)] = -np.inf  # long rows only: no row is masked throughout
    x = torch.from_numpy(x_np).to(dev)
    a, rm, rsum = _softmax(L, torch, dev, pl, x)
    want = gso.edge_softmax_np(x_np, keys, n)
    assert np.isfinite(want).all() and np.abs(a.cpu().numpy() - want).max() <= 1e-13 * np.abs(want).max()
    assert np.all(rm.cpu().numpy()[lens == 0] == -np.inf) and np.all(rsum.cpu().numpy()[lens == 0] == 0)
    g_np = W.upstream(r, c)
    g = torch.from_numpy(g_np).to(dev)
    dx, _ = _backward(L, torch, dev, pl, a, g)
    want_dx = gso.edge_softmax_backward_np(a.cpu().numpy(), g_np, keys, n)
    assert np.abs(dx.cpu().numpy() - want_dx).max() <= 1e-13 * np.abs(want_dx).max()
    assert torch.equal(_softmax(L, torch, dev, pl, x)[0], a) and torch.equal(_backward(L, torch, dev, pl, a, g)[0], dx)
    assert landmarks(M, N)["hub_col"] == int(np.argmax(np.bincount(c)))
