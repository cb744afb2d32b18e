"""GIN, GINE and edge-ReLU aggregation on the GPU on one rank.  The kernels hnh_edge_relu_aggregate_step_f64 / _grad_f64 /
_edge_grad_f64 against numpy at every table width, at odd widths and past 256 (column windows), on normal and integer
inputs (X_v + E_i == 0 exactly, for the strict mask), at odd leading dimensions and misaligned rows, past one resident
wave, on the skewed graph's hub rows, with the sums carried across two blocks, and bit-identical repeats.  The op
Distributed_Sparse::edgeReluAggregate / edgeReluAggregateBackward at p = 1 under every algorithm; the model's forward,
input gradient and every parameter gradient against tests/gin_oracle.py's literal per-edge GINConv / GINEConv;
train_step, link_train_step and graph_train_step against a torch AdamW loop; an untrained eps under weight decay; the
handle checks; two learning checks; refusals."""
import ctypes as C

import numpy as np
import pytest
import torch

from distributed_sddmm_b200 import driver as D
from distributed_sddmm_b200 import lib
from oracle import hnh_oracle as orc
from tests import gin_oracle as go
from tests import graph_readout_oracle as gro
from tests.skewed_graph import skewed_tuples
from tests.test_graph_sage_gpu import _dev_rows, _host_rows, _st, inputs
from tests.test_link_prediction_gpu import csr_block

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
SEED = 0xC0FFEE + 427
ALGS = ["15d_fusion1", "15d_fusion2", "15d_sparse", "25d_dense_replicate", "25d_sparse_replicate"]
WIDTHS = [1, 3, 4, 8, 16, 32, 64, 100, 128, 256, 257, 602]


@pytest.fixture(scope="module")
def world():
    D.world_init("self")
    yield
    D.world_finalize()


# ---- the kernels --------------------------------------------------------------------------------------------------------
def _ptrs(rowStart, col_idx):
    return torch.from_numpy(rowStart).to(DEV), torch.from_numpy(col_idx).to(DEV)


def run_step(rowStart, col_idx, X, E, A0, ld=(None, None, None), offset=0):
    n, f = A0.shape
    ldx, lde, lda = (l or f for l in ld)
    xb, eb, ab = _dev_rows(X, ldx, offset), _dev_rows(E, lde, offset), _dev_rows(A0, lda, offset)
    rs, ci = _ptrs(rowStart, col_idx)
    p = lambda b: b.data_ptr() + 8 * offset  # noqa: E731
    rc = lib().hnh_edge_relu_aggregate_step_f64(rs.data_ptr(), ci.data_ptr(), n, len(col_idx), p(xb), ldx, p(eb), lde, f, p(ab), lda,
                                                _st())
    assert rc == 0, lib().hnh_last_error_string()
    torch.cuda.synchronize()
    return _host_rows(ab, n, f, lda, offset)


def run_grad(rowStart, col_idx, X, E, dA, dX0, ld=(None, None, None, None), offset=0):
    n, f = X.shape
    ldx, lde, ldd, lddx = (l or f for l in ld)
    xb, eb, db, ob = _dev_rows(X, ldx, offset), _dev_rows(E, lde, offset), _dev_rows(dA, ldd, offset), _dev_rows(dX0, lddx, offset)
    rs, ci = _ptrs(rowStart, col_idx)
    p = lambda b: b.data_ptr() + 8 * offset  # noqa: E731
    rc = lib().hnh_edge_relu_aggregate_grad_f64(rs.data_ptr(), ci.data_ptr(), n, len(col_idx), p(xb), ldx, p(eb), lde, p(db), ldd, f,
                                                p(ob), lddx, _st())
    assert rc == 0, lib().hnh_last_error_string()
    torch.cuda.synchronize()
    return _host_rows(ob, n, f, lddx, offset)


def run_edge_grad(rowStart, col_idx, dA, X, E, ld=(None, None, None, None), offset=0):
    n, f = dA.shape
    ldd, ldx, lde, ldde = (l or f for l in ld)
    db, xb, eb = _dev_rows(dA, ldd, offset), _dev_rows(X, ldx, offset), _dev_rows(E, lde, offset)
    ob = _dev_rows(np.full(E.shape, np.nan), ldde, offset)
    rs, ci = _ptrs(rowStart, col_idx)
    p = lambda b: b.data_ptr() + 8 * offset  # noqa: E731
    rc = lib().hnh_edge_relu_aggregate_edge_grad_f64(rs.data_ptr(), ci.data_ptr(), n, len(col_idx), p(db), ldd, p(xb), ldx, p(eb), lde,
                                                     f, p(ob), ldde, _st())
    assert rc == 0, lib().hnh_last_error_string()
    torch.cuda.synchronize()
    return _host_rows(ob, len(col_idx), f, ldde, offset)


def close(got, want, tol):
    return np.abs(got - want).max() <= tol * max(np.abs(want).max(), 1.0)


def check_kernels(rowStart, col_idx, X, E, ld_step=(None,) * 3, ld_grad=(None,) * 4, ld_edge=(None,) * 4, offset=0):
    """The step from zeros, the same over two blocks carrying the sums, the dX and dE kernels, against numpy."""
    n, f = len(rowStart) - 1, X.shape[1]
    rows = np.repeat(np.arange(n), np.diff(rowStart))
    want = go.edge_relu_aggregate(rows, col_idx, n, X, E)
    A = run_step(rowStart, col_idx, X, E, np.zeros((n, f)), ld_step, offset)
    assert close(A, want, 1e-13)
    # two blocks: the first half of every row's entries, then the rest, carrying the sums (as ring steps do)
    k = np.arange(len(col_idx)) - rowStart[rows]
    first = k < np.diff(rowStart)[rows] // 2
    starts = [np.searchsorted(rows[m], np.arange(n + 1)).astype(np.int64) for m in (first, ~first)]
    A1 = run_step(starts[0], col_idx[first], X, E[first], np.zeros((n, f)), ld_step, offset)
    A2 = run_step(starts[1], col_idx[~first], X, E[~first], A1, ld_step, offset)
    assert close(A2, want, 1e-13)
    dA = np.random.default_rng(f + 2).standard_normal((n, f))
    refX, refE = go.edge_relu_aggregate_backward(rows, col_idx, X, E, dA, X.shape[0])
    # dX on the transposed block (the rows of X are its stored rows; E follows its entries)
    order = np.lexsort((rows, col_idx))
    tr, tc = col_idx[order], rows[order]
    tStart = np.searchsorted(tr, np.arange(X.shape[0] + 1)).astype(np.int64)
    dX0 = np.random.default_rng(f + 3).standard_normal(X.shape)
    dX = run_grad(tStart, tc, X, E[order], dA, dX0, ld_grad, offset)
    assert close(dX, dX0 + refX, 1e-12)
    dE = run_edge_grad(rowStart, col_idx, dA, X, E, ld_edge, offset)
    assert np.array_equal(dE, refE)
    # bit-identical repeats
    assert np.array_equal(run_grad(tStart, tc, X, E[order], dA, dX0, ld_grad, offset), dX)
    assert np.array_equal(run_step(rowStart, col_idx, X, E, np.zeros((n, f)), ld_step, offset), A)
    return X[col_idx] + E


@pytest.mark.parametrize("kind", ["normal", "int"])
@pytest.mark.parametrize("f", WIDTHS)
def test_kernels_match_numpy(world, f, kind):
    rng = np.random.default_rng(SEED + f)
    rowStart, col_idx = csr_block(rng, 300, 300)  # empty rows, duplicates, a hub row of 150 entries
    X = inputs(rng, 300, f, kind)
    E = inputs(rng, len(col_idx), f, kind)
    s = check_kernels(rowStart, col_idx, X, E)
    if kind == "int":
        assert (s == 0).any()  # the strict mask was exercised


@pytest.mark.parametrize("f", [4, 64, 256, 5, 602])
def test_kernels_odd_ld_and_misaligned_rows(world, f):
    rng = np.random.default_rng(SEED + 2 * f)
    rowStart, col_idx = csr_block(rng, 200, 200)
    X, E = inputs(rng, 200, f, "int"), inputs(rng, len(col_idx), f, "int")
    o = f + 1
    for lds, ldg, lde, offset in (((o, f, f), (o, f, f, f), (f, o, f, f), 0), ((f, o, f), (f, o, f, f), (f, f, o, f), 0),
                                  ((f, f, o), (f, f, o, f), (f, f, f, o), 0), ((f, f, f), (f, f, f, o), (o, f, f, f), 0),
                                  ((f, f, f), (f, f, f, f), (f, f, f, f), 1)):
        check_kernels(rowStart, col_idx, X, E, lds, ldg, lde, offset)


@pytest.mark.parametrize("f,n", [(4, 200000), (64, 30000), (256, 12000), (5, 40000)])
def test_kernels_past_one_wave(world, f, n):
    rng = np.random.default_rng(SEED + n)
    rowStart, col_idx = csr_block(rng, n, n, per_row=3)
    check_kernels(rowStart, col_idx, inputs(rng, n, f, "int"), inputs(rng, len(col_idx), f, "int"))


@pytest.mark.parametrize("f", [64, 7])
def test_kernels_on_the_skewed_graph(world, f):
    rows, cols = skewed_tuples(4200, 4200, SEED)
    rows, cols = rows.astype(np.int64), cols.astype(np.int64)
    order = np.lexsort((cols, rows))
    rows, cols = rows[order], cols[order]
    rowStart = np.searchsorted(rows, np.arange(4201)).astype(np.int64)
    rng = np.random.default_rng(SEED + f)
    check_kernels(rowStart, cols, inputs(rng, 4200, f, "normal"), inputs(rng, len(cols), f, "normal"))


def test_gin_combine_kernels(world):
    rng = np.random.default_rng(SEED + 1)
    n = 100003
    M, X, dH = (torch.from_numpy(rng.standard_normal(n)).to(DEV) for _ in range(3))
    eps = torch.tensor([0.375], dtype=torch.float64, device=DEV)
    H, dX, deps = torch.empty_like(M), torch.empty_like(M), torch.empty(1, dtype=torch.float64, device=DEV)
    assert lib().hnh_gin_combine_f64(H.data_ptr(), M.data_ptr(), X.data_ptr(), eps.data_ptr(), n, _st()) == 0
    assert lib().hnh_gin_combine_grad_f64(dX.data_ptr(), deps.data_ptr(), dH.data_ptr(), X.data_ptr(), eps.data_ptr(), n, _st()) == 0
    torch.cuda.synchronize()
    assert torch.allclose(H, M + 1.375 * X, rtol=1e-15, atol=1e-15) and torch.equal(dX, 1.375 * dH)
    assert abs(float(deps) - float((dH * X).sum())) <= 1e-12 * n
    first = float(deps)
    assert lib().hnh_gin_combine_grad_f64(dX.data_ptr(), deps.data_ptr(), dH.data_ptr(), X.data_ptr(), eps.data_ptr(), n, _st()) == 0
    torch.cuda.synchronize()
    assert float(deps) == first  # bit-identical repeats


# ---- the op at p = 1 ----------------------------------------------------------------------------------------------------
def op_case(alg_name, f, logM=7, npr=5):
    N = 1 << logM
    rows, cols, _ = orc.er_tuples(logM, npr, SEED + f)
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    rows, cols = np.append(rows, [3, 3, 3]), np.append(cols, [cols[0]] * 3)  # duplicates
    keep = rows != 9  # an empty row
    rows, cols = rows[keep], cols[keep]
    S = D.SpmatLocal.from_tuples(N, N, rows, cols, np.ones(len(rows)))
    alg = D.Algorithm(alg_name, S, 8, 1)
    X = inputs(np.random.default_rng(SEED + 5), N, f, "int")
    return N, rows, cols, alg, X


def dense_of(a):
    d = D.Dense.create(*a.shape)
    d.from_host(a)
    return d


@pytest.mark.parametrize("f", [8, 64, 13, 300])
@pytest.mark.parametrize("alg_name", ALGS)
def test_edge_relu_aggregate_op(world, alg_name, f):
    N, rows, cols, alg, X = op_case(alg_name, f)
    nA, nB = alg.like_A_matrix().shape[0], alg.like_B_matrix().shape[0]
    Xh = np.zeros((nB, f))
    Xh[:N] = X
    Xd = dense_of(Xh)
    EA, EB = (dense_of(go.edge_rows(*alg.entry_coordinates(m), f)) for m in ("A", "B"))
    A = D.Dense.create(nA, f, 7.0)
    alg.edge_relu_aggregate(Xd, EA, A)
    E = go.edge_rows(rows, cols, f)
    assert (X[cols] + E == 0).any()
    want = go.edge_relu_aggregate(rows, cols, N, X, E)
    got = A.to_host()
    assert close(got[:N], want, 1e-13)
    assert not got[9].any() and not got[N:].any()  # the empty row and the padding
    dAh = np.zeros((nA, f))
    dAh[:N] = np.random.default_rng(SEED + 6).standard_normal((N, f))
    dA, dX, dE = dense_of(dAh), D.Dense.create(nB, f, 3.0), D.Dense.create(0, 0)
    refX, refE = go.edge_relu_aggregate_backward(rows, cols, X, E, dAh[:N], N)
    alg.edge_relu_aggregate_backward(Xd, EA, EB, dA, dX)
    assert close(dX.to_host()[:N], refX, 1e-12)
    alg.edge_relu_aggregate_backward(Xd, EA, EB, dA, dX, dE, accumulate=True)
    assert close(dX.to_host()[:N], 2 * refX, 1e-12)
    ra, ca = alg.entry_coordinates("A")
    mine = go.edge_relu_aggregate_backward(ra, ca, X, go.edge_rows(ra, ca, f), dAh[:N], N)[1]
    assert dE.shape == (len(ra), f) and np.array_equal(dE.to_host(), mine)
    A2 = D.Dense.create(nA, f)
    alg.edge_relu_aggregate(Xd, EA, A2)
    assert np.array_equal(A2.to_host(), got)


def test_edge_relu_aggregate_refusals(world):
    N, rows, cols, alg, X = op_case("15d_fusion1", 8)
    nA, nB = alg.like_A_matrix().shape[0], alg.like_B_matrix().shape[0]
    nE, nEB = len(alg.like_S_values()), len(alg.like_ST_values())
    Xd, EA, EB = D.Dense.create(nB, 8), D.Dense.create(nE, 8), D.Dense.create(nEB, 8)
    A, dA, dX, dE = D.Dense.create(nA, 8), D.Dense.create(nA, 8), D.Dense.create(nB, 8), D.Dense.create(nE, 8)
    for args, msg in (((Xd, EA, Xd), "another operand|A-shaped"), ((Xd, EA, EA), "A-shaped"), ((D.Dense.create(nB, 0), EA, A), "width"),
                      ((Xd, EA, D.Dense.create(nA, 7)), "A-shaped"), ((D.Dense.create(nB + 1, 8), EA, A), "like_B_matrix"),
                      ((Xd, D.Dense.create(nE + 1, 8), A), "E_A is"), ((Xd, D.Dense.create(nE, 9), A), "E_A is")):
        with pytest.raises(RuntimeError, match=msg):
            alg.edge_relu_aggregate(*args)
    for args, msg in (((Xd, EA, None, dA, dX), "both orders"), ((Xd, None, EB, dA, dX), "both orders"),
                      ((Xd, EA, EB, dA, Xd), "another operand"), ((Xd, EA, EB, dA, dA), "another operand"),
                      ((Xd, EA, EB, dA, D.Dense.create(nB, 9)), "dX is"), ((Xd, EA, D.Dense.create(nEB + 1, 8), dA, dX), "E_B is"),
                      ((Xd, EA, EB, dA, dX, EA), "another operand"), ((Xd, EA, EB, dA, dX, dX), "another operand"),
                      ((Xd, EA, EB, dA, dX, dA), "another operand")):
        with pytest.raises(RuntimeError, match=msg):
            alg.edge_relu_aggregate_backward(*args)
    alg.edge_relu_aggregate_backward(Xd, EA, EB, dA, dX, dE)  # the shapes that are right run


# ---- the model ----------------------------------------------------------------------------------------------------------
LAYER_SETS = {1: [(6, 9, 4)], 2: [(6, 10, 8), (8, 7, 3)], 3: [(6, 10, 8), (8, 12, 5), (5, 6, 4)]}


def set_params(net, params):
    for l, P in enumerate(params):
        for name, v in P.items():
            net.set_param(l, name, v)


def build(layers, edge_dim=0, train_eps=True, logM=7, npr=5, alg_name="15d_fusion1", pattern=None, seed=SEED):
    N = 1 << logM
    if pattern is None:
        rows, cols, _ = orc.er_tuples(logM, npr, seed)
    else:
        rows, cols = pattern
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    S = D.SpmatLocal.from_tuples(N, N, rows, cols, np.ones(len(rows)))
    alg = D.Algorithm(alg_name, S, layers[0][0], 1)
    net = D.GIN(alg, layers, edge_dim=edge_dim, eps=0.5, train_eps=train_eps)
    rng = np.random.default_rng(seed + 1)
    params = go.random_params(layers, edge_dim, rng)
    set_params(net, params)
    if edge_dim:
        net.set_edge_attributes(go.attr_of(*alg.entry_coordinates("A"), edge_dim), go.attr_of(*alg.entry_coordinates("B"), edge_dim))
    X = rng.uniform(-1, 1, (N, layers[0][0]))
    Xl = np.zeros(net.buffer_shape(0))
    Xl[:N] = X
    net.set_input(Xl)
    shape = net.buffer_shape(len(layers))
    G = np.zeros(shape)
    G[:N] = rng.uniform(-1, 1, (N, shape[1]))
    attr = go.attr_of(rows, cols, edge_dim) if edge_dim else None
    return dict(N=N, rows=rows, cols=cols, alg=alg, net=net, params=params, X=X, G=G, layers=layers, attr=attr, train_eps=train_eps)


def rel_err(got, ref):
    return np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-300)


def check_against_model(P, tol=1e-9):
    net, N, layers = P["net"], P["N"], P["layers"]
    net.forward()
    out, dX, dP = go.forward_backward(P["rows"], P["cols"], N, layers, P["params"], P["X"], P["G"][:N], P["attr"])
    assert np.abs(out).max() > 0
    assert rel_err(net.buffer(len(layers))[:N], out) < tol
    net.backward(P["G"])
    assert rel_err(net.input_grad()[:N], dX) < tol
    for l, grads in enumerate(dP):
        for name, g in grads.items():
            got = net.param_grad(l, name)
            assert got.shape == g.shape, (l, name)
            if name == "eps" and not P["train_eps"]:
                assert not got.any()  # a constant: its gradient reads 0
            else:
                assert rel_err(got, g) < tol, (l, name, rel_err(got, g))


@pytest.mark.parametrize("train_eps", [True, False])
@pytest.mark.parametrize("edge_dim", [0, 3])
@pytest.mark.parametrize("n_layers", [1, 2, 3])
def test_model_matches_oracle(world, n_layers, edge_dim, train_eps):
    check_against_model(build(LAYER_SETS[n_layers], edge_dim, train_eps))


@pytest.mark.parametrize("edge_dim", [0, 2])
@pytest.mark.parametrize("alg_name", ALGS)
def test_model_on_every_algorithm_with_duplicates_and_empty_rows(world, alg_name, edge_dim):
    rng = np.random.default_rng(SEED + 9)
    N = 128
    rows, cols = rng.integers(0, N, 500), rng.integers(0, N, 500)
    rows[rows % 7 == 0] = 1  # rows without entries and a hub row
    rows[:5], cols[:5] = 2, 11  # duplicates
    check_against_model(build([(6, 16, 16), (16, 8, 3)], edge_dim, alg_name=alg_name, pattern=(rows, cols)))


def test_wide_layers(world):
    check_against_model(build([(300, 64, 16), (16, 300, 4)], 4, logM=8))


def test_gine_state_dict_through_param(world):
    """A GINEConv's state dict, loaded through set_param, gives the oracle's output and gradients."""
    from tests.test_gin import _GINEConv
    P = build([(6, 10, 8)], 3)
    net, N = P["net"], P["N"]
    conv = _GINEConv(6, 10, 8, 3)
    torch.manual_seed(SEED)
    with torch.no_grad():
        conv.eps.fill_(0.2)
    sd = {k: v.detach().numpy() for k, v in conv.state_dict().items()}
    mine = {"lin1": sd["nn.0.weight"].T, "lin1_bias": sd["nn.0.bias"], "lin2": sd["nn.2.weight"].T, "lin2_bias": sd["nn.2.bias"],
            "edge": sd["lin.weight"].T, "edge_bias": sd["lin.bias"], "eps": sd["eps"]}
    set_params(net, [mine])
    P["params"] = [mine]
    check_against_model(P)


def test_backward_repeats_bit_identical_and_needs_a_forward(world):
    P = build(LAYER_SETS[2], 2)
    net = P["net"]
    net.forward()
    net.backward(P["G"])
    first = [net.param_grad(l, n) for l in range(2) for n in net.param_names()] + [net.input_grad()]
    net.forward()
    net.backward(P["G"])
    again = [net.param_grad(l, n) for l in range(2) for n in net.param_names()] + [net.input_grad()]
    assert all(np.array_equal(a, b) for a, b in zip(first, again))
    net.set_param(0, "eps", [0.0])
    with pytest.raises(RuntimeError, match="no forward pass"):
        net.backward(P["G"])
    net.forward()
    net.set_edge_attributes(go.attr_of(*P["alg"].entry_coordinates("A"), 2), go.attr_of(*P["alg"].entry_coordinates("B"), 2))
    with pytest.raises(RuntimeError, match="no forward pass"):
        net.backward(P["G"])


def test_model_refusals(world):
    P = build(LAYER_SETS[1], 0)
    alg, net = P["alg"], P["net"]
    out = C.c_void_p()
    flat = (C.c_int * 3)(6, 9, 4)
    assert lib().hnhd_gin_create(alg.h, 1, flat, -1, 0.0, 0, C.byref(out)) == -1 and b"edge_dim" in lib().hnh_last_error_string()
    for eps in (float("nan"), float("inf")):
        assert lib().hnhd_gin_create(alg.h, 1, flat, 0, eps, 0, C.byref(out)) == -1 and b"eps" in lib().hnh_last_error_string()
    with pytest.raises(RuntimeError, match="does not take the width"):
        net2 = (C.c_int * 6)(6, 9, 4, 5, 3, 2)
        D.check(lib().hnhd_gin_create(alg.h, 2, net2, 0, 0.0, 0, C.byref(out)), "gin_create")
    with pytest.raises(RuntimeError, match="sizes must be positive"):
        D.GIN(alg, [(6, 0, 4)])
    with pytest.raises(RuntimeError, match="no parameter"):
        net.param_shape(0, "edge")
    with pytest.raises(RuntimeError, match="no such layer"):
        net.param(1, "lin1")
    with pytest.raises(RuntimeError, match="no dropout"):
        net._forward(0.1, 0)
    with pytest.raises(ValueError, match="no edge features"):
        net.set_edge_attributes(np.zeros((2, 1)), np.zeros((2, 1)))
    assert net.param_shape(0, "lin1") == (6, 9) and net.param_shape(0, "lin2") == (9, 4) and net.param_shape(0, "eps") == (1,)
    assert net.param(0, "eps").tolist() == [0.25]
    edged = D.GIN(alg, [(6, 9, 4)], edge_dim=2)
    assert edged.param(0, "eps").tolist() == [0.0] and not edged.param(0, "lin1").any()
    assert edged.param_shape(0, "edge") == (2, 6) and edged.param_shape(0, "edge_bias") == (6,)
    with pytest.raises(RuntimeError, match="no edge attributes"):
        edged.forward()
    nA, nB = len(alg.like_S_values()), len(alg.like_ST_values())
    with pytest.raises(RuntimeError, match="edge attributes for"):
        edged.set_edge_attributes(np.zeros((nA + 1, 2)), np.zeros((nB, 2)))


def test_handles_are_refused_by_other_models_calls(world):
    P = build(LAYER_SETS[1], 2)
    gin, alg = P["net"], P["alg"]
    p = (C.c_double * 4)()
    assert lib().hnhd_gt_set_edge_attributes(gin.h, p, 0, p, 0) == -1
    assert b"takes a graph transformer model, not a GIN one" in lib().hnh_last_error_string()
    assert lib().hnhd_gat_set_attention(gin.h, b"softmax") == -1 and b"takes a GAT model" in lib().hnh_last_error_string()
    assert lib().hnhd_gat_weight_shape(gin.h, 0, 0, None, None) == -1
    gt = D.GraphTransformer(alg, [(6, 2, 2)], edge_dim=2)
    assert lib().hnhd_gin_set_edge_attributes(gt.h, p, 0, p, 0) == -1
    assert b"takes a GIN model, not a graph transformer one" in lib().hnh_last_error_string()


# ---- training -----------------------------------------------------------------------------------------------------------
def node_labels(net, N, seed):
    rng = np.random.default_rng(seed)
    labels = rng.integers(0, 3, N)
    labels[rng.random(N) < 0.3] = -1
    lab = np.full(net.buffer_shape(len(net.layers))[0], -1)
    lab[:N] = labels
    return labels, D.NodeLabels(net, lab, 3)


def check_trained(net, trained):
    for l, Pt in enumerate(trained):
        for k, v in Pt.items():
            assert close(net.param(l, k), v, 1e-9), (l, k)


@pytest.mark.parametrize("train_eps", [True, False])
@pytest.mark.parametrize("edge_dim", [0, 3])
def test_train_step_matches_torch_adamw(world, edge_dim, train_eps):
    P = build([(6, 10, 8), (8, 7, 3)], edge_dim, train_eps)
    N, net = P["N"], P["net"]
    labels, L = node_labels(net, N, SEED + 11)
    opt = D.AdamW(lr=1e-2, max_grad_norm=0.5)
    got = [net.train_step(L, opt) for _ in range(4)]
    res, trained = go.train(P["rows"], P["cols"], N, P["layers"], P["params"], P["X"], labels, 4, attr=P["attr"], train_eps=train_eps,
                            lr=1e-2, max_grad_norm=0.5)
    for g, w in zip(got, res):
        assert abs(g.loss - w[0]) <= 1e-9 * abs(w[0]) and abs(g.grad_norm - w[3]) <= 1e-9 * abs(w[3])
        assert (g.correct, g.labelled) == (w[1], w[2])
    check_trained(net, trained)


def test_untrained_eps_is_unchanged_by_weight_decay(world):
    P = build([(6, 10, 8), (8, 7, 3)], 2, train_eps=False)
    net = P["net"]
    before = [net.param(l, "eps") for l in range(2)]
    _, L = node_labels(net, P["N"], SEED + 12)
    opt = D.AdamW(lr=0.1, weight_decay=0.5)
    for _ in range(3):
        net.train_step(L, opt)
    assert all(np.array_equal(net.param(l, "eps"), b) for l, b in enumerate(before))
    assert not np.array_equal(net.param(0, "lin1"), P["params"][0]["lin1"])


@pytest.mark.parametrize("edge_dim", [0, 2])
def test_link_train_step_matches_torch_adamw(world, edge_dim):
    P = build([(6, 10, 8), (8, 7, 4)], edge_dim)
    N = P["N"]
    rng = np.random.default_rng(SEED + 12)
    tr, tc = rng.integers(0, N, 4 * N), rng.integers(0, N, 4 * N)
    y = rng.choice([0.0, 1.0], 4 * N)
    algT = D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, tr, tc, y), 6, 1)
    t = D.LinkTargets(P["net"], algT)
    opt = D.AdamW(lr=1e-2)
    got = [P["net"].link_train_step(t, opt) for _ in range(3)]
    res, trained = go.train_link(P["rows"], P["cols"], N, P["layers"], P["params"], P["X"], (tr, tc, y), 3, attr=P["attr"], lr=1e-2)
    for g, w in zip(got, res):
        assert abs(g.loss - w[0]) <= 1e-9 * abs(w[0]) and abs(g.grad_norm - w[3]) <= 1e-9 * abs(w[3])
        assert g.labelled == w[2] and abs(g.correct - w[1]) <= 1
    check_trained(P["net"], trained)


@pytest.mark.parametrize("edge_dim", [0, 2])
@pytest.mark.parametrize("pool", gro.POOLS)
def test_graph_train_step_matches_torch_adamw(world, pool, edge_dim):
    P = build([(6, 10, 8), (8, 7, 4)], edge_dim)
    N, net = P["N"], P["net"]
    rng = np.random.default_rng(SEED + 13)
    G = 9
    batch = np.full(net.buffer_shape(2)[0], -1, np.int64)
    batch[:N] = rng.integers(0, G, N)
    batch[:N][rng.random(N) < 0.1] = -1
    ro = D.GraphReadout(net, batch, G, pool=pool, num_classes=3)
    W, b = rng.uniform(-1, 1, (4, 3)), rng.uniform(-0.5, 0.5, 3)
    ro.set_param("weight", W)
    ro.set_param("bias", b)
    labels = rng.integers(0, 3, G)
    labels[1] = -1
    gl = D.GraphLabels(ro, labels, 3)
    opt = D.AdamW(lr=1e-2, max_grad_norm=0.5)
    got = [net.graph_train_step(ro, gl, opt) for _ in range(3)]
    tp = go._leaves(P["params"])
    x, a = go._t(P["X"]), None if P["attr"] is None else go._t(P["attr"])
    want, head = gro.train(lambda t: go.model_torch(P["rows"], P["cols"], N, P["layers"], tp, x, a), go._trained(tp), batch[:N], G,
                           pool, (W, b), labels, 3, lr=1e-2, max_grad_norm=0.5)
    for g, w in zip(got, want):
        assert abs(g.loss - w[0]) <= 1e-9 * abs(w[0]) and abs(g.grad_norm - w[3]) <= 1e-9 * abs(w[3]), (g, w)
        assert (g.correct, g.labelled) == (w[1], w[2])
    check_trained(net, [{k: v.detach().numpy() for k, v in Pd.items()} for Pd in tp])
    assert close(ro.param("weight"), head[0], 1e-9) and close(ro.param("bias"), head[1], 1e-9)


# ---- learning checks ----------------------------------------------------------------------------------------------------
def random_init(net, rng):
    for l in range(len(net.layers)):
        for name in net.param_names():
            if name == "eps":
                continue
            shape = net.param_shape(l, name)
            net.set_param(l, name, rng.uniform(-1, 1, shape) / np.sqrt(shape[0]))


def regular_batch(G, n, seed):
    """G graphs of n nodes each, half 2-regular (a cycle) and half 3-regular (a cycle with its diameters), both edge
    directions stored; label 1 for the 3-regular ones."""
    rng = np.random.default_rng(seed)
    labels = np.repeat([0, 1], G // 2)
    rng.shuffle(labels)
    rows, cols = [], []
    for g in range(G):
        base = g * n
        for i in range(n):
            nbrs = [(i + 1) % n, (i - 1) % n] + ([(i + n // 2) % n] if labels[g] else [])
            rows += [base + i] * len(nbrs)
            cols += [base + j for j in nbrs]
    return G * n, np.array(rows), np.array(cols), np.repeat(np.arange(G), n), labels


def train_graphs(net, N, batch, labels, G, steps, lr=1e-2):
    Xl = np.zeros(net.buffer_shape(0))
    Xl[:N] = 1.0  # constant node features
    net.set_input(Xl)
    b = np.full(net.buffer_shape(len(net.layers))[0], -1, np.int64)
    b[:N] = batch
    ro = D.GraphReadout(net, b, G, pool="mean", num_classes=2)
    gl = D.GraphLabels(ro, labels, 2)
    opt = D.AdamW(lr=lr)
    steps = [net.graph_train_step(ro, gl, opt) for _ in range(steps)]
    return steps, net.graph_evaluate(ro, gl)[3]


@pytest.mark.parametrize("model", ["gin", "sage_mean"])
def test_learning_regular_graphs(world, model):
    """GIN separates 2-regular from 3-regular graphs under a mean readout; GraphSAGE-mean sees the same rows in both."""
    G, n = 32, 12
    N, rows, cols, batch, labels = regular_batch(G, n, SEED + 14)
    alg = D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, rows, cols, np.ones(len(rows))), 1, 1)
    net = D.GIN(alg, [(1, 16, 16), (16, 16, 8)]) if model == "gin" else D.GraphSAGE(alg, [(1, 16), (16, 8)], aggr="mean")
    random_init(net, np.random.default_rng(SEED + 15))
    steps, logits = train_graphs(net, N, batch, labels, G, 150)
    if model == "gin":
        assert steps[-1].loss < 0.5 * steps[0].loss and steps[-1].correct >= 0.9 * G, (steps[0], steps[-1])
    else:  # every node row is the same in both kinds of graph: no better than the balanced prior
        assert np.abs(logits - logits[0]).max() <= 1e-12 * max(np.abs(logits).max(), 1.0)
        assert steps[-1].correct <= G // 2


@pytest.mark.parametrize("edge_dim", [1, 0])
def test_learning_a_label_carried_by_edge_attributes(world, edge_dim):
    """Cycles of one shape whose edges carry +1 (label 1) or -1 (label 0): GINE learns the label, GIN cannot."""
    G, n = 32, 10
    rng = np.random.default_rng(SEED + 16)
    labels = np.repeat([0, 1], G // 2)
    rng.shuffle(labels)
    rows = np.concatenate([[g * n + i, g * n + i] for g in range(G) for i in range(n)])
    cols = np.concatenate([[g * n + (i + 1) % n, g * n + (i - 1) % n] for g in range(G) for i in range(n)])
    N = G * n
    alg = D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, rows, cols, np.ones(len(rows))), 1, 1)
    net = D.GIN(alg, [(1, 16, 16), (16, 16, 8)], edge_dim=edge_dim)
    random_init(net, np.random.default_rng(SEED + 17))
    if edge_dim:
        sign = lambda r: (2.0 * labels[np.asarray(r, np.int64) // n] - 1.0)[:, None]  # noqa: E731
        ra, _ = alg.entry_coordinates("A")
        rb, _ = alg.entry_coordinates("B")
        net.set_edge_attributes(sign(ra), sign(rb))
    steps, logits = train_graphs(net, N, np.repeat(np.arange(G), n), labels, G, 150)
    if edge_dim:
        assert steps[-1].loss < 0.5 * steps[0].loss and steps[-1].correct >= 0.9 * G, (steps[0], steps[-1])
    else:
        assert np.abs(logits - logits[0]).max() <= 1e-12 * max(np.abs(logits).max(), 1.0)
        assert steps[-1].correct <= G // 2
