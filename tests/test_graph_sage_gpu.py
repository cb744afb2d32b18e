"""GraphSAGE and max aggregation on the GPU on one rank.  The kernels hnh_max_aggregate_step_f64 / _grad_f64 against
numpy at every table width, at odd widths and past 256 (column windows), at odd leading dimensions and misaligned rows,
with empty rows, hub rows, duplicates, integer-valued and ReLU'd inputs (heavy ties), more rows than one resident wave,
and bit-identical repeats.  The op Distributed_Sparse::maxAggregate / maxAggregateBackward at p = 1 under every
algorithm; the model's forward, backward and parameter gradients against tests/graph_sage_oracle.py for each
aggregator; train_step and link_train_step against a torch AdamW loop; refusals.  Multi-rank cases are in
tests/test_graph_sage_multirank_gpu.py."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from distributed_sddmm_b200 import driver as D
from distributed_sddmm_b200 import lib
from oracle import hnh_oracle as orc
from tests import graph_sage_oracle as gso
from tests.skewed_graph import skewed_tuples
from tests.test_link_prediction_gpu import csr_block

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
SEED = 0xC0FFEE + 191
ALGS = ["15d_fusion1", "15d_fusion2", "15d_sparse", "25d_dense_replicate", "25d_sparse_replicate"]


@pytest.fixture(scope="module")
def world():
    D.world_init("self")
    yield
    D.world_finalize()


def _st():
    return torch.cuda.current_stream().cuda_stream


# ---- the kernels --------------------------------------------------------------------------------------------------------
def _dev_rows(A, ld, offset):
    """A (rows x f) as a device buffer with leading dimension ld, starting `offset` doubles in; NaN elsewhere."""
    n, f = A.shape
    buf = torch.full((offset + max(n * ld, 1) + 1,), math.nan, dtype=torch.float64, device=DEV)
    if n:
        buf[offset:offset + n * ld].view(n, ld)[:, :f] = torch.from_numpy(np.ascontiguousarray(A)).to(DEV)
    return buf


def _host_rows(buf, n, f, ld, offset):
    d = buf[offset:offset + n * ld].view(n, ld)
    if ld > f:
        assert torch.isnan(d[:, f:]).all()  # the columns past f are not written
    return d[:, :f].cpu().numpy()


def run_step(rowStart, col_idx, X, Z0, C0, ld=(None, None, None), offset=0):
    """One step kernel on (Z0, C0); returns (Z, C)."""
    n, f = Z0.shape
    ldx, ldz, ldc = (l or f for l in ld)
    xb, zb, cb = _dev_rows(X, ldx, offset), _dev_rows(Z0, ldz, offset), _dev_rows(C0, ldc, offset)
    rs, ci = torch.from_numpy(rowStart).to(DEV), torch.from_numpy(col_idx).to(DEV)
    p = lambda b: b.data_ptr() + 8 * offset  # noqa: E731
    rc = lib().hnh_max_aggregate_step_f64(rs.data_ptr(), ci.data_ptr(), n, len(col_idx), p(xb), ldx, f, p(zb), ldz, p(cb), ldc, _st())
    assert rc == 0, lib().hnh_last_error_string()
    torch.cuda.synchronize()
    return _host_rows(zb, n, f, ldz, offset), _host_rows(cb, n, f, ldc, offset)


def run_grad(rowStart, col_idx, X, Z, G, dX0, ld=(None, None, None, None), offset=0):
    n, f = X.shape
    ldx, ldz, ldg, lddx = (l or f for l in ld)
    xb, zb, gb, db = _dev_rows(X, ldx, offset), _dev_rows(Z, ldz, offset), _dev_rows(G, ldg, offset), _dev_rows(dX0, lddx, offset)
    rs, ci = torch.from_numpy(rowStart).to(DEV), torch.from_numpy(col_idx).to(DEV)
    p = lambda b: b.data_ptr() + 8 * offset  # noqa: E731
    rc = lib().hnh_max_aggregate_grad_f64(rs.data_ptr(), ci.data_ptr(), n, len(col_idx), p(xb), ldx, p(zb), ldz, p(gb), ldg, f,
                                          p(db), lddx, _st())
    assert rc == 0, lib().hnh_last_error_string()
    torch.cuda.synchronize()
    return _host_rows(db, n, f, lddx, offset)


def inputs(rng, n, f, kind):
    if kind == "int":
        return rng.integers(-3, 4, (n, f)).astype(np.float64)
    X = rng.standard_normal((n, f))
    return np.maximum(X, 0.0) if kind == "relu" else X


def check_kernels(rowStart, col_idx, X, ld_step=(None, None, None), ld_grad=(None, None, None, None), offset=0):
    """The step from (-inf, 0) and a merge into a pre-filled state, the finish, and the grad, against numpy."""
    n, f = len(rowStart) - 1, X.shape[1]
    rows = np.repeat(np.arange(n), np.diff(rowStart))
    # from the initial state
    Z, Cn = run_step(rowStart, col_idx, X, np.full((n, f), -np.inf), np.zeros((n, f)), ld_step, offset)
    wZ, wC = gso.max_aggregate(rows, col_idx, n, X)
    empty = np.diff(rowStart) == 0
    assert np.array_equal(Cn, wC) and np.isneginf(Z[empty]).all()
    assert np.array_equal(np.where(wC == 0, 0.0, Z), wZ)
    # merging into a state that holds an earlier block's maxima (ties with it add their counts)
    Z0 = np.where(np.random.default_rng(f).random((n, f)) < 0.5, wZ, wZ - 1.0)
    C0 = np.random.default_rng(f + 1).integers(1, 4, (n, f)).astype(np.float64)
    Z1, C1 = run_step(rowStart, col_idx, X, Z0, C0, ld_step, offset)
    m = ~empty[:, None] & np.ones((1, f), bool)
    wZ1 = np.where(m, np.maximum(Z0, wZ), Z0)
    wC1 = np.where(m, np.where(Z0 > wZ, C0, np.where(Z0 == wZ, C0 + wC, wC)), C0)
    assert np.array_equal(Z1, wZ1) and np.array_equal(C1, wC1)
    # grad: dX += sum_u [X_v == Z_u] G_u, on the transposed block (the rows of X are its stored rows)
    dZ = np.random.default_rng(f + 2).standard_normal((n, f))
    G = np.divide(dZ, wC, out=np.zeros_like(dZ), where=wC != 0)
    order = np.lexsort((rows, col_idx))
    tr, tc = col_idx[order], rows[order]
    Xm = X  # the block is square: X's rows are its columns
    tStart = np.searchsorted(tr, np.arange(Xm.shape[0] + 1)).astype(np.int64)
    dX0 = np.random.default_rng(f + 3).standard_normal(Xm.shape)
    dX = run_grad(tStart, tc, Xm, wZ, G, dX0, ld_grad, offset)
    want = dX0 + gso.max_aggregate_backward(rows, col_idx, wZ, wC, dZ, Xm.shape[0], Xm)
    assert np.abs(dX - want).max() <= 1e-13 * max(np.abs(want).max(), 1.0)
    again = run_grad(tStart, tc, Xm, wZ, G, dX0, ld_grad, offset)
    assert np.array_equal(again, dX)  # bit-identical repeats
    assert np.array_equal(run_step(rowStart, col_idx, X, Z0, C0, ld_step, offset)[0], Z1)
    return wC


WIDTHS = [1, 3, 4, 8, 16, 32, 64, 100, 128, 256, 257, 602]


@pytest.mark.parametrize("kind", ["normal", "relu", "int"])
@pytest.mark.parametrize("f", WIDTHS)
def test_max_kernels_match_numpy(world, f, kind):
    rng = np.random.default_rng(SEED + f)
    rowStart, col_idx = csr_block(rng, 300, 300)  # empty rows, duplicates, a hub row of 150 entries
    C = check_kernels(rowStart, col_idx, inputs(rng, 300, f, kind))
    if kind != "normal":
        assert C.max() > 1  # ties happened


@pytest.mark.parametrize("f", [4, 64, 256, 5, 602])
def test_max_kernels_odd_ld_and_misaligned_rows(world, f):
    rng = np.random.default_rng(SEED + 2 * f)
    rowStart, col_idx = csr_block(rng, 200, 200)
    X = inputs(rng, 200, f, "relu")
    for lds, ldg, offset in (((f + 1, f, f), (f + 1, f, f, f), 0), ((f, f + 1, f), (f, f + 1, f, f), 0),
                             ((f, f, f + 1), (f, f, f + 1, f + 1), 0), ((f, f, f), (f, f, f, f), 1)):
        check_kernels(rowStart, col_idx, X, lds, ldg, offset)


@pytest.mark.parametrize("f,n", [(4, 200000), (64, 30000), (256, 12000), (5, 40000)])
def test_max_kernels_past_one_wave(world, f, n):
    rng = np.random.default_rng(SEED + n)
    rowStart, col_idx = csr_block(rng, n, n, per_row=3)
    check_kernels(rowStart, col_idx, inputs(rng, n, f, "int"))


@pytest.mark.parametrize("f", [64, 7])
def test_max_kernels_on_the_skewed_graph(world, f):
    rows, cols = skewed_tuples(4200, 4200, SEED)
    rows, cols = rows.astype(np.int64), cols.astype(np.int64)
    order = np.lexsort((cols, rows))
    rows, cols = rows[order], cols[order]
    rowStart = np.searchsorted(rows, np.arange(4201)).astype(np.int64)
    check_kernels(rowStart, cols, inputs(np.random.default_rng(SEED + f), 4200, f, "relu"))


def test_finish_and_grad_scale(world):
    Z = torch.tensor([-math.inf, 2.0, -math.inf, 0.5], dtype=torch.float64, device=DEV)
    Cn = torch.tensor([0.0, 1.0, 0.0, 3.0], dtype=torch.float64, device=DEV)
    assert lib().hnh_max_aggregate_finish_f64(Z.data_ptr(), Cn.data_ptr(), 4, _st()) == 0
    dZ = torch.tensor([5.0, 2.0, 7.0, 3.0], dtype=torch.float64, device=DEV)
    G = torch.empty(4, dtype=torch.float64, device=DEV)
    assert lib().hnh_max_aggregate_grad_scale_f64(G.data_ptr(), dZ.data_ptr(), Cn.data_ptr(), 4, _st()) == 0
    torch.cuda.synchronize()
    assert Z.tolist() == [0.0, 2.0, 0.0, 0.5] and G.tolist() == [0.0, 2.0, 0.0, 1.0]


# ---- the op at p = 1 ----------------------------------------------------------------------------------------------------
def op_case(alg_name, f, kind, logM=7, npr=5):
    N = 1 << logM
    rows, cols, _ = orc.er_tuples(logM, npr, SEED + f)
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    rows, cols = np.append(rows, [3, 3, 3]), np.append(cols, [cols[0]] * 3)  # duplicates
    keep = rows != 9  # an empty row
    rows, cols = rows[keep], cols[keep]
    S = D.SpmatLocal.from_tuples(N, N, rows, cols, np.ones(len(rows)))
    alg = D.Algorithm(alg_name, S, 8, 1)
    X = inputs(np.random.default_rng(SEED + 5), N, f, kind)
    return N, rows, cols, alg, X


@pytest.mark.parametrize("f", [8, 64, 13, 300])
@pytest.mark.parametrize("alg_name", ALGS)
def test_max_aggregate_op(world, alg_name, f):
    N, rows, cols, alg, X = op_case(alg_name, f, "relu")
    nA, nB = alg.like_A_matrix().shape[0], alg.like_B_matrix().shape[0]
    Xd, Z, Cd = D.Dense.create(nB, f), D.Dense.create(nA, f, 7.0), D.Dense.create(nA, f, 7.0)
    Xh = np.zeros((nB, f))
    Xh[:N] = X
    Xd.from_host(Xh)
    alg.max_aggregate(Xd, Z, Cd)
    wZ, wC = gso.max_aggregate(rows, cols, N, X)
    assert np.array_equal(Z.to_host()[:N], wZ) and np.array_equal(Cd.to_host()[:N], wC)
    assert not Cd.to_host()[9].any() and not Z.to_host()[9].any()  # the empty row
    dZh = np.zeros((nA, f))
    dZh[:N] = np.random.default_rng(SEED + 6).standard_normal((N, f))
    dZ, dX = D.Dense.create(nA, f), D.Dense.create(nB, f, 3.0)
    dZ.from_host(dZh)
    want = gso.max_aggregate_backward(rows, cols, wZ, wC, dZh[:N], N, X)
    alg.max_aggregate_backward(Xd, Z, Cd, dZ, dX)
    got = dX.to_host()
    assert np.abs(got[:N] - want).max() <= 1e-13 * np.abs(want).max()
    alg.max_aggregate_backward(Xd, Z, Cd, dZ, dX, accumulate=True)
    assert np.abs(dX.to_host()[:N] - 2 * want).max() <= 1e-13 * np.abs(want).max()
    Z2, C2 = D.Dense.create(nA, f), D.Dense.create(nA, f)
    alg.max_aggregate(Xd, Z2, C2)
    assert np.array_equal(Z2.to_host(), Z.to_host()) and np.array_equal(C2.to_host(), Cd.to_host())


def test_max_aggregate_refusals(world):
    N, rows, cols, alg, X = op_case("15d_fusion1", 8, "normal")
    nA, nB = alg.like_A_matrix().shape[0], alg.like_B_matrix().shape[0]
    Xd, Z, Cd, dZ, dX = (D.Dense.create(n, 8) for n in (nB, nA, nA, nA, nB))
    for args, msg in (((Xd, Z, Z), "another operand"), ((Xd, Xd, Cd), "another operand"),
                      ((D.Dense.create(nB, 0), Z, Cd), "width must be positive"), ((Xd, D.Dense.create(nA, 9), Cd), "A-shaped"),
                      ((D.Dense.create(nB + 1, 8), Z, Cd), "like_B_matrix")):
        with pytest.raises(RuntimeError, match=msg):
            alg.max_aggregate(*args)
    with pytest.raises(RuntimeError, match="another operand"):
        alg.max_aggregate_backward(Xd, Z, Cd, dZ, dZ)
    with pytest.raises(RuntimeError, match="dX is"):
        alg.max_aggregate_backward(Xd, Z, Cd, dZ, D.Dense.create(nB, 9))


# ---- the model ----------------------------------------------------------------------------------------------------------
def build(layers, aggr, logM=7, npr=5, alg_name="15d_fusion1", pattern=None, seed=SEED):
    N = 1 << logM
    if pattern is None:
        rows, cols, _ = orc.er_tuples(logM, npr, seed)
    else:
        rows, cols = pattern
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    S = D.SpmatLocal.from_tuples(N, N, rows, cols, np.ones(len(rows)))
    alg = D.Algorithm(alg_name, S, layers[0][0], 1)
    net = D.GraphSAGE(alg, layers, aggr=aggr)
    rng = np.random.default_rng(seed + 1)
    params = gso.random_params(layers, rng)
    for l, P in enumerate(params):
        for name, v in P.items():
            net.set_param(l, name, v)
    X = rng.uniform(-1, 1, (N, layers[0][0]))
    Xl = np.zeros(net.buffer_shape(0))
    Xl[:N] = X
    net.set_input(Xl)
    shape = net.buffer_shape(len(layers))
    G = np.zeros(shape)
    G[:N] = rng.uniform(-1, 1, (N, shape[1]))
    return dict(N=N, rows=rows, cols=cols, S=S, alg=alg, net=net, params=params, X=X, G=G, layers=layers, aggr=aggr)


def rel_err(got, ref):
    return np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-300)


def check_against_model(P):
    net, N, layers = P["net"], P["N"], P["layers"]
    net.forward()
    out, dX, dP = gso.forward_backward(P["rows"], P["cols"], N, layers, P["params"], P["X"], P["aggr"], P["G"][:N])
    assert np.abs(out).max() > 0
    assert rel_err(net.buffer(len(layers))[:N], out) < 1e-12
    net.backward(P["G"])
    assert rel_err(net.input_grad()[:N], dX) < 1e-11
    for l, grads in enumerate(dP):
        for name, g in grads.items():
            got = net.param_grad(l, name)
            assert got.shape == g.shape, (l, name)
            assert rel_err(got, g) < 1e-11, (l, name, rel_err(got, g))


LAYER_SETS = {1: [(6, 4)], 2: [(6, 8), (8, 3)], 3: [(6, 8), (8, 5), (5, 4)]}


@pytest.mark.parametrize("aggr", gso.AGGREGATIONS)
@pytest.mark.parametrize("n_layers", [1, 2, 3])
def test_model_matches_oracle(world, n_layers, aggr):
    check_against_model(build(LAYER_SETS[n_layers], aggr))


@pytest.mark.parametrize("aggr", gso.AGGREGATIONS)
@pytest.mark.parametrize("alg_name", ALGS)
def test_model_on_every_algorithm_with_duplicates_and_empty_rows(world, alg_name, aggr):
    rng = np.random.default_rng(SEED + 9)
    N = 128
    rows, cols = rng.integers(0, N, 500), rng.integers(0, N, 500)
    rows[rows % 7 == 0] = 1  # rows without entries and a hub row
    rows[:5], cols[:5] = 2, 11  # duplicates
    check_against_model(build([(6, 64), (64, 3)], aggr, alg_name=alg_name, pattern=(rows, cols)))


@pytest.mark.parametrize("aggr", gso.AGGREGATIONS)
def test_wide_input_layer(world, aggr):
    check_against_model(build([(602, 16), (16, 4)], aggr, logM=8))


def test_backward_repeats_bit_identical_and_needs_a_forward(world):
    P = build(LAYER_SETS[2], "max")
    net = P["net"]
    net.forward()
    net.backward(P["G"])
    first = [net.param_grad(l, n) for l in range(2) for n in net.param_names()] + [net.input_grad()]
    net.forward()
    net.backward(P["G"])
    again = [net.param_grad(l, n) for l in range(2) for n in net.param_names()] + [net.input_grad()]
    assert all(np.array_equal(a, b) for a, b in zip(first, again))
    net.set_param(0, "root", P["params"][0]["root"])
    with pytest.raises(RuntimeError, match="no forward pass"):
        net.backward(P["G"])
    net.forward()
    net.set_input(np.zeros(net.buffer_shape(0)))
    with pytest.raises(RuntimeError, match="no forward pass"):
        net.backward(P["G"])


def test_model_refusals(world):
    P = build(LAYER_SETS[1], "mean")
    alg = P["alg"]
    out = C.c_void_p()
    flat = (C.c_int * 2)(6, 4)
    assert lib().hnhd_sage_create(alg.h, 1, flat, b"lstm", C.byref(out)) == -1
    assert b"unknown aggregation" in lib().hnh_last_error_string()
    with pytest.raises(RuntimeError, match="does not take the width"):
        D.GraphSAGE(alg, [(6, 4), (5, 3)])
    with pytest.raises(RuntimeError, match="sizes must be positive"):
        D.GraphSAGE(alg, [(6, 0)])
    with pytest.raises(RuntimeError, match="no parameter"):
        P["net"].param_shape(0, "query")
    with pytest.raises(RuntimeError, match="no such layer"):
        P["net"].param(1, "root")
    assert P["net"].param_shape(0, "neigh") == (6, 4) and P["net"].param_shape(0, "neigh_bias") == (4,)


# ---- training -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("aggr", gso.AGGREGATIONS)
def test_train_step_matches_torch_adamw(world, aggr):
    P = build([(6, 8), (8, 3)], aggr)
    N = P["N"]
    rng = np.random.default_rng(SEED + 11)
    labels = rng.integers(0, 3, N)
    labels[rng.random(N) < 0.3] = -1
    lab = np.full(P["net"].buffer_shape(2)[0], -1)
    lab[:N] = labels
    L = D.NodeLabels(P["net"], lab, 3)
    opt = D.AdamW(lr=1e-2, max_grad_norm=0.5)
    got = [P["net"].train_step(L, opt) for _ in range(5)]
    res, trained = gso.train(P["rows"], P["cols"], N, P["layers"], P["params"], P["X"], aggr, labels, 5, lr=1e-2,
                             max_grad_norm=0.5)
    for g, w in zip(got, res):
        assert abs(g.loss - w[0]) <= 1e-10 * abs(w[0]) and abs(g.grad_norm - w[3]) <= 1e-10 * abs(w[3])
        assert (g.correct, g.labelled) == (w[1], w[2])
    for l, Pt in enumerate(trained):
        for k, v in Pt.items():
            assert np.abs(P["net"].param(l, k) - v).max() <= 1e-9 * max(np.abs(v).max(), 1.0), (l, k)


@pytest.mark.parametrize("aggr", gso.AGGREGATIONS)
def test_link_train_step_matches_torch_adamw(world, aggr):
    P = build([(6, 8), (8, 4)], aggr)
    N = P["N"]
    rng = np.random.default_rng(SEED + 12)
    tr, tc = rng.integers(0, N, 4 * N), rng.integers(0, N, 4 * N)
    y = rng.choice([0.0, 1.0], 4 * N)
    algT = D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, tr, tc, y), 6, 1)
    t = D.LinkTargets(P["net"], algT)
    opt = D.AdamW(lr=1e-2)
    got = [P["net"].link_train_step(t, opt) for _ in range(4)]
    res, trained = gso.train_link(P["rows"], P["cols"], N, P["layers"], P["params"], P["X"], aggr, (tr, tc, y), 4, lr=1e-2)
    for g, w in zip(got, res):
        assert abs(g.loss - w[0]) <= 1e-10 * abs(w[0]) and abs(g.grad_norm - w[3]) <= 1e-10 * abs(w[3])
        assert g.labelled == w[2] and abs(g.correct - w[1]) <= 1
    for l, Pt in enumerate(trained):
        for k, v in Pt.items():
            assert np.abs(P["net"].param(l, k) - v).max() <= 1e-9 * max(np.abs(v).max(), 1.0), (l, k)
    loss, correct, count, scores = P["net"].link_evaluate(t)
    H = P["net"].buffer(2)[:N]
    assert (H < 0).any()  # the last layer has no ReLU
    er, ec = algT.entry_coordinates("A")
    want = (H[er] * H[ec]).sum(1)
    assert count == 4 * N and np.abs(scores - want).max() <= 1e-12 * np.abs(want).max()
