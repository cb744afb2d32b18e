"""Graph-level prediction on the GPU on one rank.  The kernels hnh_segment_pool_f64 / hnh_segment_pool_grad_f64 against
numpy at every table width and at odd widths, at odd leading dimensions, with empty graphs, 1-node graphs, one graph
of most rows, graphs crossing chunk boundaries, unsorted ids, rows in no graph, all rows in no graph, and max ties
(duplicated rows, -0.0 / +0.0); bit-identical repeats.  GraphReadout.pool / pool_backward, graph_train_step for GAT,
the graph transformer (with dropout), GraphSAGE and R-GCN under each pool with and without the head, graph_evaluate's
logits, the refusals, and a learning check.  Multi-rank cases are in tests/test_graph_readout_multirank_gpu.py."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from distributed_sddmm_b200 import driver as D
from distributed_sddmm_b200 import lib
from oracle import hnh_oracle as orc
from tests import gat_backward_oracle as gbk
from tests import graph_readout_oracle as gro
from tests import graph_sage_oracle as gso
from tests import graph_transformer_oracle as gto
from tests import rgcn_oracle as rgo

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
SEED = 0xC0FFEE + 401
TABLE = [4, 8, 16, 32, 64, 128, 256]
ODD = [1, 3, 6, 33, 100, 300]


@pytest.fixture(scope="module")
def world():
    D.world_init("self")
    yield
    D.world_finalize()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _d(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


# ---- the kernels --------------------------------------------------------------------------------------------------------
def batches(rng, n):
    """name -> (batch, G) over n rows"""
    mixed = rng.integers(0, 40, n)
    mixed[rng.random(n) < 0.1] = -1
    mixed[mixed == 7] = 8  # an empty graph
    mixed[5] = 40  # a 1-node graph
    big = np.where(rng.random(n) < 0.8, 0, rng.integers(1, 6, n))  # one graph of most rows, unsorted
    runs = np.repeat(np.arange(n // 300 + 1), 300)[:n]  # sorted, contiguous, each crossing a chunk boundary
    return {"mixed": (mixed, 42), "big": (big, 6), "runs": (runs, int(runs.max()) + 1), "none": (np.full(n, -1), 3)}


def run_pool(H, batch, G, pool, ldh=None, ldp=None):
    n, r = H.shape
    ldh, ldp = ldh or r, ldp or r
    seg_start, seg_rows, chunk_first, chunk_seg = (_d(a) for a in gro.plan(batch, G))
    hb = torch.full((max(n, 1), ldh), math.nan, dtype=torch.float64, device=DEV)
    hb[:n, :r] = _d(H)
    P = torch.full((G, ldp), math.nan, dtype=torch.float64, device=DEV)
    Cb = torch.full((G, ldp), math.nan, dtype=torch.float64, device=DEV) if pool == "max" else None
    chunks = len(chunk_seg)
    nb = lib().hnh_segment_pool_workspace_bytes(chunks, r, int(pool == "max"))
    ws = torch.empty(max(nb // 8, 1), dtype=torch.float64, device=DEV)
    rc = lib().hnh_segment_pool_f64(seg_start.data_ptr(), seg_rows.data_ptr(), chunk_first.data_ptr(), chunk_seg.data_ptr(), G, chunks,
                                    hb.data_ptr(), ldh, r, P.data_ptr(), ldp, Cb.data_ptr() if Cb is not None else None, ldp,
                                    ws.data_ptr(), nb, _st())
    assert rc == 0, lib().hnh_last_error_string()
    torch.cuda.synchronize()
    if ldp > r:
        assert torch.isnan(P[:, r:]).all()
    out = P[:, :r].cpu().numpy()
    return (out, Cb[:, :r].cpu().numpy()) if Cb is not None else out


def run_grad(batch, G, dP, scale=None, H=None, P=None, Cn=None, ld=None):
    r = dP.shape[1]
    ld = ld or r
    n = len(batch)
    pad = lambda A, rows: torch.nn.functional.pad(_d(A), (0, ld - r)) if A is not None else None  # noqa: E731
    rg = _d(np.asarray(batch, np.int32))
    dPd, Hd, Pd, Cd = pad(dP, G), pad(H, n), pad(P, G), pad(Cn, G)
    sd = _d(scale) if scale is not None else None
    dH = torch.full((n, ld), math.nan, dtype=torch.float64, device=DEV)
    p = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    rc = lib().hnh_segment_pool_grad_f64(rg.data_ptr(), n, G, dPd.data_ptr(), ld, p(sd), p(Hd), ld, p(Pd), ld, p(Cd), ld, r,
                                         dH.data_ptr(), ld, _st())
    assert rc == 0, lib().hnh_last_error_string()
    torch.cuda.synchronize()
    if ld > r:
        assert torch.isnan(dH[:, r:]).all()
    return dH[:, :r].cpu().numpy()


def rel_err(got, ref):
    return np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-300)


def check_kernels(H, batch, G, ldh=None, ldp=None):
    r = H.shape[1]
    rng = np.random.default_rng(r)
    P = run_pool(H, batch, G, "sum", ldh, ldp)
    assert rel_err(P, gro.pool_np(H, batch, G, "sum")) < 1e-13
    Pm, Cm = run_pool(H, batch, G, "max", ldh, ldp)
    Pw, Cw = gro.pool_np(H, batch, G, "max")
    assert np.array_equal(Pm, Pw) and np.array_equal(Cm, Cw)
    dP = rng.standard_normal((G, r))
    scale = rng.uniform(0.5, 2.0, G)
    assert np.array_equal(run_grad(batch, G, dP, ld=ldp), gro.pool_grad_np(batch, G, dP))
    assert np.array_equal(run_grad(batch, G, dP, scale=scale, ld=ldp), gro.pool_grad_np(batch, G, dP, scale))
    Pf = np.where(Cw == 0, 0.0, Pw)
    assert np.array_equal(run_grad(batch, G, dP, H=H, P=Pf, Cn=Cw, ld=ldp), gro.pool_grad_np(batch, G, dP, H=H, P=Pf, C=Cw))


@pytest.mark.parametrize("name", ["mixed", "big", "runs", "none"])
@pytest.mark.parametrize("r", TABLE + ODD)
def test_kernels_match_numpy(world, r, name):
    rng = np.random.default_rng(SEED + r)
    n = 1500
    batch, G = batches(rng, n)[name]
    check_kernels(rng.standard_normal((n, r)), batch, G)


@pytest.mark.parametrize("r", [8, 64, 128, 5])
def test_kernels_with_ties_and_signed_zeros(world, r):
    rng = np.random.default_rng(SEED + 2 * r)
    n = 1200
    batch, G = batches(rng, n)["big"]
    H = np.round(rng.uniform(-2, 2, (n, r)))  # heavy ties, -0.0 and +0.0 among them
    H[rng.random((n, r)) < 0.2] = -0.0
    H[10] = H[11]  # duplicated rows
    check_kernels(H, batch, G)


@pytest.mark.parametrize("r", [64, 128, 7])
def test_kernels_at_odd_leading_dimensions(world, r):
    rng = np.random.default_rng(SEED + 3 * r)
    batch, G = batches(rng, 900)["mixed"]
    check_kernels(rng.standard_normal((900, r)), batch, G, ldh=r + 1, ldp=r + 3)


@pytest.mark.parametrize("r", [128, 33])
def test_kernels_repeat_bit_identically_past_one_merge_pass(world, r):
    """A graph of about 4000 rows: 16 chunks, so every merge warp combines more than one chunk partial."""
    rng = np.random.default_rng(SEED + 5)
    batch, G = batches(rng, 5000)["big"]
    assert np.bincount(batch[batch >= 0]).max() > 8 * gro.CHUNK
    H = rng.standard_normal((5000, r))
    a, b = run_pool(H, batch, G, "sum"), run_pool(H, batch, G, "sum")
    assert np.array_equal(a, b)
    assert all(np.array_equal(x, y) for x, y in zip(run_pool(H, batch, G, "max"), run_pool(H, batch, G, "max")))
    check_kernels(H, batch, G)


# ---- the models ---------------------------------------------------------------------------------------------------------
N, F0 = 128, 6


def _graph(seed=SEED):
    rows, cols, _ = orc.er_tuples(7, 5, seed)
    return np.asarray(rows, np.int64), np.asarray(cols, np.int64)


def _batch(rng, rows_local, G=9):
    b = rng.integers(0, G, N)
    b[rng.random(N) < 0.1] = -1
    b[b == 3] = 4  # an empty graph
    out = np.full(rows_local, -1, np.int64)
    out[:N] = b
    return out, G


def build(kind, pool, head, alg_name="15d_fusion1"):
    """(net, torch forward(leaves, t, dropout), leaves, getters) for one model kind on the same graph and input."""
    rows, cols = _graph()
    rng = np.random.default_rng(SEED + 7)
    X = rng.uniform(-1, 1, (N, F0))
    if kind == "rgcn":
        R = 3
        rels = rgo.hashed_relations(rows, cols, N, R)
        S = D.SpmatLocal.from_tuples(N, N, rows, cols, rels.astype(np.float64))
    else:
        S = D.SpmatLocal.from_tuples(N, N, rows, cols, np.ones(len(rows)))
    alg = D.Algorithm(alg_name, S, F0, 1)
    x = gso._t(X)
    if kind == "sage":
        layers = [(F0, 8), (8, 4)]
        net = D.GraphSAGE(alg, layers, aggr="mean")
        params = gso.random_params(layers, rng)
        fwd = lambda tp, t: gso.model_torch(rows, cols, N, layers, tp, x, "mean")  # noqa: E731
    elif kind == "rgcn":
        layers = [(F0, 8), (8, 4)]
        net = D.RGCN(alg, layers, R, aggr="sum")
        params = rgo.random_params(layers, R, rng)
        fwd = lambda tp, t: rgo.model_torch(rows, cols, rels, N, layers, tp, x, R, "sum")  # noqa: E731
    elif kind == "gt":
        layers = [(F0, 4, 2), (8, 2, 2)]
        net = D.GraphTransformer(alg, layers)
        params = gto.random_params(layers, 0, False, rng)
        fwd = lambda tp, t: gto.model_torch(rows, cols, N, layers, tp, x, None, False, 0.2, 11 + t)  # noqa: E731
    else:
        layers = [(F0, 4, 2), (8, 4, 1)]
        net = D.GAT(alg, layers)
        weights = [[rng.uniform(-1, 1, (f, d)) / math.sqrt(f) for _ in range(H)] for f, d, H in layers]
        for l, (f, d, H) in enumerate(layers):
            for h in range(H):
                net.set_weight(l, h, weights[l][h])
        ri, ci = gbk.edges(rows, cols, N)
        params = [{f"w{h}": w for h, w in enumerate(ws)} for ws in weights]
        fwd = lambda tp, t: gbk.gat_forward_torch(ri, ci, N, layers, [[P[f"w{h}"] for h in range(len(P))] for P in tp], 0.2, x)  # noqa: E731
    if kind != "gat":
        for l, P in enumerate(params):
            for k, v in P.items():
                net.set_param(l, k, v)
    net.set_input(np.vstack([X, np.zeros((net.buffer_shape(0)[0] - N, F0))]))
    r = net.buffer_shape(len(layers))[1]
    batch, G = _batch(rng, net.buffer_shape(len(layers))[0])
    Cc = 3 if head else r
    ro = D.GraphReadout(net, batch, G, pool=pool, num_classes=Cc if head else None)
    W = b = None
    if head:
        W, b = rng.uniform(-1, 1, (r, Cc)), rng.uniform(-0.5, 0.5, Cc)
        ro.set_param("weight", W)
        ro.set_param("bias", b)
    labels = rng.integers(0, Cc, G)
    labels[1] = -1
    evalf = (lambda tp: gto.model_torch(rows, cols, N, layers, tp, x)) if kind == "gt" else (lambda tp: fwd(tp, 0))  # noqa: E731
    return dict(net=net, alg=alg, ro=ro, fwd=fwd, evalf=evalf, params=params, batch=batch[:N], G=G, C=Cc, head=(W, b) if head else None,
                labels=labels, layers=layers, kind=kind)


def _close(got, want, tol):
    return np.abs(got - want).max() <= tol * max(np.abs(want).max(), 1.0)


CASES = [(k, p, h) for k in ("sage", "rgcn", "gt", "gat") for p in gro.POOLS for h in (True, False)]


@pytest.mark.parametrize("kind,pool,head", CASES)
def test_graph_train_step_matches_torch(world, kind, pool, head):
    B = build(kind, pool, head)
    net, ro, steps = B["net"], B["ro"], 3
    labels = D.GraphLabels(ro, B["labels"], B["C"])
    opt = D.AdamW(lr=1e-2, max_grad_norm=0.5)
    dropout = 0.2 if kind == "gt" else 0.0
    got = [net.graph_train_step(ro, labels, opt, dropout, 11 + t) if kind == "gt" else net.graph_train_step(ro, labels, opt)
           for t in range(steps)]
    tp = [{k: gso._t(v).clone().requires_grad_() for k, v in P.items()} for P in B["params"]]
    want, trained_head = gro.train(lambda t: B["fwd"](tp, t), [v for P in tp for v in P.values()], B["batch"], B["G"], pool,
                                   B["head"], B["labels"], steps, lr=1e-2, max_grad_norm=0.5)
    for t, (g, w) in enumerate(zip(got, want)):
        assert abs(g.loss - w[0]) <= 1e-9 * abs(w[0]) and abs(g.grad_norm - w[3]) <= 1e-9 * abs(w[3]), (t, g, w)
        assert (g.correct, g.labelled) == (w[1], w[2]), (t, g, w)
    for l, P in enumerate(tp):
        for k, v in P.items():
            got_v = net.weight(l, int(k[1:])) if kind == "gat" else net.param(l, k)
            assert _close(got_v, v.detach().numpy(), 1e-9), (l, k)
    if head:
        assert _close(ro.param("weight"), trained_head[0], 1e-9) and _close(ro.param("bias"), trained_head[1], 1e-9)
        assert ro.param_grad("weight").shape == trained_head[0].shape
    loss, correct, labelled, logits = net.graph_evaluate(ro, labels)
    H = B["evalf"]([{k: v.detach() for k, v in P.items()} for P in tp])
    hl = None if not head else tuple(gso._t(v) for v in (ro.param("weight"), ro.param("bias")))
    want_logits = gro.head_torch(gro.pool_torch(H, B["batch"], B["G"], pool), hl).numpy()
    assert _close(logits, want_logits, 1e-10) and labelled == int((B["labels"] >= 0).sum())


@pytest.mark.parametrize("pool", gro.POOLS)
def test_pool_and_pool_backward_on_dense(world, pool):
    B = build("sage", pool, False)
    net, ro = B["net"], B["ro"]
    net.forward()
    Hh = net.buffer(2)
    H = D.Dense.create(*Hh.shape)
    H.from_host(Hh)
    P = ro.pool(H)
    Ht = gso._t(Hh[:N]).requires_grad_()
    want = gro.pool_torch(Ht, B["batch"], B["G"], pool)
    assert _close(P.to_host(), want.detach().numpy(), 1e-13)
    dPh = np.random.default_rng(3).standard_normal(want.shape)
    dP = D.Dense.create(*dPh.shape)
    dP.from_host(dPh)
    dH = ro.pool_backward(dP).to_host()
    want.backward(gso._t(dPh))
    assert _close(dH[:N], Ht.grad.numpy(), 1e-13) and not dH[N:].any()
    again = ro.pool(H).to_host()
    assert np.array_equal(again, P.to_host())


def test_refusals(world):
    B = build("sage", "mean", True)
    net, ro = B["net"], B["ro"]
    rows_local = net.buffer_shape(2)[0]
    ok = np.full(rows_local, -1, np.int64)
    ok[:N] = 0
    for batch, G, msg in ((ok[:-1], 2, "ids for"), (np.where(ok == 0, 5, ok), 2, "not below"), (ok, 0, "G must")):
        with pytest.raises(RuntimeError, match=msg):
            D.GraphReadout(net, batch, G)
    with pytest.raises(RuntimeError, match="classes"):
        D.GraphLabels(D.GraphReadout(net, ok, 2), np.zeros(2, np.int64), 3)  # no head: the logits are 4 wide
    if rows_local > N:
        bad = ok.copy()
        bad[-1] = 0
        with pytest.raises(RuntimeError, match="padding row"):
            D.GraphReadout(net, bad, 2, num_classes=3)
    out = C.c_void_p()
    assert lib().hnhd_readout_create(net.h, ok.ctypes.data, len(ok), 2, b"attention", 0, C.byref(out)) == -1
    assert b"unknown pool" in lib().hnh_last_error_string()
    assert lib().hnhd_readout_create(net.h, ok.ctypes.data, len(ok), 2, b"sum", -1, C.byref(out)) == -1
    assert lib().hnhd_readout_create(net.h, ok.ctypes.data, len(ok), 1 << 31, b"sum", 3, C.byref(out)) == -1
    with pytest.raises(RuntimeError, match="labels for"):
        D.GraphLabels(ro, np.zeros(B["G"] + 1, np.int64), 3)
    with pytest.raises(RuntimeError, match="not below"):
        D.GraphLabels(ro, np.full(B["G"], 3), 3)
    with pytest.raises(RuntimeError, match="classes"):
        D.GraphLabels(ro, np.zeros(B["G"], np.int64), 4)
    with pytest.raises(RuntimeError, match="no parameter"):
        ro.param_shape("query")
    assert ro.param_shape("weight") == (4, 3) and ro.param_shape("bias") == (3,)
    labels = D.GraphLabels(ro, B["labels"], 3)
    other = build("sage", "mean", True)
    with pytest.raises(RuntimeError, match="another model"):
        other["net"].graph_train_step(ro, labels, D.AdamW())
    with pytest.raises(RuntimeError, match="another readout"):
        other["net"].graph_train_step(other["ro"], labels, D.AdamW())
    opt = D.AdamW()
    net.train_step(D.NodeLabels(net, np.full(rows_local, -1), 4), opt)  # the optimizer now holds the model's spans alone
    with pytest.raises(RuntimeError, match="not those of the optimizer"):
        net.graph_train_step(ro, labels, opt)
    with pytest.raises(RuntimeError, match="no parameter"):
        D.GraphReadout(net, ok, 2).param_shape("weight")  # no head
    with pytest.raises(RuntimeError, match="dropout"):
        net._graph_train_step(ro, labels, D.AdamW(), 0.1, 0)
    S = D.SpmatLocal.from_tuples(N, N, *_graph(), np.ones(len(_graph()[0])))
    sparse = D.GraphSAGE(D.Algorithm("15d_sparse", S, F0, 1), [(F0, 4)])
    rs = sparse.buffer_shape(1)[0]
    b = np.full(rs, -1, np.int64)
    b[:min(N, rs)] = 0
    D.GraphReadout(sparse, b, 1)  # p = 1: every layout holds full rows


def test_learning_graph_sizes(world):
    """GraphSAGE-sum with a sum readout on constant inputs learns labels = [n_g > 6] to train accuracy 1.0."""
    rng = np.random.default_rng(SEED + 9)
    sizes = rng.integers(2, 12, 24)
    G, n = len(sizes), int(sizes.sum())
    batch = np.repeat(np.arange(G), sizes)
    rows, cols = [], []
    start = 0
    for s in sizes:  # a ring inside every graph
        u = np.arange(start, start + s)
        rows += list(u)
        cols += list(np.roll(u, 1))
        start += s
    S = D.SpmatLocal.from_tuples(n, n, np.array(rows), np.array(cols), np.ones(len(rows)))
    net = D.GraphSAGE(D.Algorithm("15d_fusion1", S, 1, 1), [(1, 8), (8, 8)], aggr="sum")
    for l, P in enumerate(gso.random_params([(1, 8), (8, 8)], rng, scale=0.5)):
        for k, v in P.items():
            net.set_param(l, k, v)
    net.set_input(np.ones(net.buffer_shape(0)))
    b = np.full(net.buffer_shape(2)[0], -1, np.int64)
    b[:n] = batch
    ro = D.GraphReadout(net, b, G, pool="sum", num_classes=2)
    y = (sizes > 6).astype(np.int64)
    labels = D.GraphLabels(ro, y, 2)
    opt = D.AdamW(lr=0.05, weight_decay=0.0)
    for _ in range(300):
        st = net.graph_train_step(ro, labels, opt)
        if st.correct == G:
            break
    assert net.graph_evaluate(ro, labels)[1] == G
