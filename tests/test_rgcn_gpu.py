"""R-GCN and relational aggregation on the GPU on one rank.  The kernels hnh_relational_aggregate_f64 / _grad_f64
against numpy at every table width, at odd widths and past 256 (column windows), at R = 1, 3 and 8 with one relation
without entries, at odd leading dimensions and misaligned rows, with empty rows, hub rows and duplicates, more rows than
one resident wave, on the skewed graph, with values that are no relation (skipped, guard cells untouched), and
bit-identical repeats; hnh_window_scale_f64 and hnh_relation_check_f64.  The op Distributed_Sparse::relationalAggregate
/ relationalAggregateBackward at p = 1 under every algorithm; the model's forward, backward and every gradient against
tests/rgcn_oracle.py; R = 1 against GraphSAGE's mean; train_step and link_train_step against a torch AdamW loop;
refusals.  Multi-rank cases are in tests/test_rgcn_multirank_gpu.py."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from distributed_sddmm_b200 import driver as D
from distributed_sddmm_b200 import lib
from oracle import hnh_oracle as orc
from tests import rgcn_oracle as ro
from tests.skewed_graph import skewed_tuples
from tests.test_link_prediction_gpu import csr_block

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
SEED = 0xC0FFEE + 241
ALGS = ["15d_fusion1", "15d_fusion2", "15d_sparse", "25d_dense_replicate", "25d_sparse_replicate"]
NOT_RELATIONS = [-1.0, None, 0.5, math.nan, math.inf, -math.inf]  # None: R


@pytest.fixture(scope="module")
def world():
    D.world_init("self")
    yield
    D.world_finalize()


def _st():
    return torch.cuda.current_stream().cuda_stream


# ---- the kernels --------------------------------------------------------------------------------------------------------
def _dev_rows(A, ld, offset):
    """A (rows x w) as a device buffer with leading dimension ld, starting `offset` doubles in; NaN elsewhere."""
    n, w = A.shape
    buf = torch.full((offset + max(n * ld, 1) + 1,), math.nan, dtype=torch.float64, device=DEV)
    if n:
        buf[offset:offset + n * ld].view(n, ld)[:, :w] = torch.from_numpy(np.ascontiguousarray(A)).to(DEV)
    return buf


def _host_rows(buf, n, w, ld, offset):
    """The rows back; every guard cell (before, between and after them) must still hold NaN."""
    flat = buf.cpu().numpy()
    d = flat[offset:offset + n * ld].reshape(n, ld)
    assert np.isnan(flat[:offset]).all() and np.isnan(flat[offset + n * ld:]).all() and np.isnan(d[:, w:]).all()
    return d[:, :w].copy()


def run_aggregate(rowStart, col_idx, vals, X, A0, R, ld=(None, None), offset=0):
    n, f = len(rowStart) - 1, X.shape[1]
    ldx, lda = ld[0] or f, ld[1] or R * f
    xb, ab = _dev_rows(X, ldx, offset), _dev_rows(A0, lda, offset)
    rs, ci, v = (torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a in (rowStart, col_idx, vals))
    p = lambda b: b.data_ptr() + 8 * offset  # noqa: E731
    rc = lib().hnh_relational_aggregate_f64(rs.data_ptr(), ci.data_ptr(), v.data_ptr(), n, len(col_idx), p(xb), ldx, f, R, p(ab),
                                            lda, _st())
    assert rc == 0, lib().hnh_last_error_string()
    torch.cuda.synchronize()
    return _host_rows(ab, n, R * f, lda, offset)


def run_grad(rowStart, col_idx, vals, dA, dX0, R, ld=(None, None), offset=0):
    n, f = len(rowStart) - 1, dX0.shape[1]
    ldda, lddx = ld[0] or R * f, ld[1] or f
    ab, xb = _dev_rows(dA, ldda, offset), _dev_rows(dX0, lddx, offset)
    rs, ci, v = (torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a in (rowStart, col_idx, vals))
    p = lambda b: b.data_ptr() + 8 * offset  # noqa: E731
    rc = lib().hnh_relational_aggregate_grad_f64(rs.data_ptr(), ci.data_ptr(), v.data_ptr(), n, len(col_idx), p(ab), ldda, f, R,
                                                 p(xb), lddx, _st())
    assert rc == 0, lib().hnh_last_error_string()
    torch.cuda.synchronize()
    return _host_rows(xb, n, f, lddx, offset)


def relations(rng, nnz, R):
    """Uniform relations, leaving relation R // 2 without entries when R > 1."""
    pool = [r for r in range(R) if R == 1 or r != R // 2]
    return rng.choice(pool, nnz).astype(np.float64)


def check_kernels(rowStart, col_idx, vals, X, R, ld_agg=(None, None), ld_grad=(None, None), offset=0):
    """The aggregate into a pre-filled A and the grad into a pre-filled dX, against numpy; repeats bit-identical."""
    n, m, f = len(rowStart) - 1, X.shape[0], X.shape[1]
    rows = np.repeat(np.arange(n), np.diff(rowStart))
    rng = np.random.default_rng(f + R)
    A0 = rng.standard_normal((n, R * f))
    A = run_aggregate(rowStart, col_idx, vals, X, A0, R, ld_agg, offset)
    want = A0 + ro.relational_aggregate(rows, col_idx, vals, n, X, R)
    assert np.abs(A - want).max() <= 1e-13 * max(np.abs(want).max(), 1.0)
    untouched = ro.relation_counts(rows, vals, n, R).repeat(f, 1) == 0
    assert np.array_equal(A[untouched], A0[untouched])  # windows without entries are not written
    assert np.array_equal(run_aggregate(rowStart, col_idx, vals, X, A0, R, ld_agg, offset), A)
    # grad: dX += sum_u dA[u, rel f ..], on the transposed block (the rows of X are its stored rows)
    order = np.lexsort((rows, col_idx))
    tr, tc, tv = col_idx[order], rows[order], vals[order]
    tStart = np.searchsorted(tr, np.arange(m + 1)).astype(np.int64)
    dA = rng.standard_normal((n, R * f))
    dX0 = rng.standard_normal((m, f))
    dX = run_grad(tStart, tc, tv, dA, dX0, R, ld_grad, offset)
    want = dX0 + ro.relational_aggregate_backward(rows, col_idx, vals, dA, m, R)
    assert np.abs(dX - want).max() <= 1e-13 * max(np.abs(want).max(), 1.0)
    assert np.array_equal(run_grad(tStart, tc, tv, dA, dX0, R, ld_grad, offset), dX)  # bit-identical repeats


WIDTHS = [1, 3, 4, 8, 16, 32, 64, 100, 128, 256, 257, 602]


@pytest.mark.parametrize("R", [1, 3, 8])
@pytest.mark.parametrize("f", WIDTHS)
def test_relational_kernels_match_numpy(world, f, R):
    rng = np.random.default_rng(SEED + f + 1000 * R)
    rowStart, col_idx = csr_block(rng, 300, 300)  # empty rows, duplicates, a hub row of 150 entries
    check_kernels(rowStart, col_idx, relations(rng, len(col_idx), R), rng.standard_normal((300, f)), R)


@pytest.mark.parametrize("f", [4, 64, 256, 5, 602])
def test_relational_kernels_odd_ld_and_misaligned_rows(world, f):
    rng = np.random.default_rng(SEED + 2 * f)
    R = 3
    rowStart, col_idx = csr_block(rng, 200, 200)
    vals = relations(rng, len(col_idx), R)
    X = rng.standard_normal((200, f))
    for ld_agg, ld_grad, offset in (((f + 1, None), (R * f + 1, None), 0), ((None, R * f + 1), (None, f + 1), 0),
                                    ((None, None), (None, None), 1)):
        check_kernels(rowStart, col_idx, vals, X, R, ld_agg, ld_grad, offset)


@pytest.mark.parametrize("f,n", [(4, 200000), (64, 30000), (256, 12000), (5, 40000)])
def test_relational_kernels_past_one_wave(world, f, n):
    rng = np.random.default_rng(SEED + n)
    rowStart, col_idx = csr_block(rng, n, n, per_row=3)
    check_kernels(rowStart, col_idx, relations(rng, len(col_idx), 4), rng.standard_normal((n, f)), 4)


@pytest.mark.parametrize("f", [64, 7])
def test_relational_kernels_on_the_skewed_graph(world, f):
    R = 5
    rows, cols = skewed_tuples(4200, 4200, SEED)
    rows, cols = rows.astype(np.int64), cols.astype(np.int64)
    vals = ro.hashed_relations(rows, cols, 4200, R)
    order = np.lexsort((cols, rows))
    rows, cols, vals = rows[order], cols[order], vals[order]
    rowStart = np.searchsorted(rows, np.arange(4201)).astype(np.int64)
    check_kernels(rowStart, cols, vals, np.random.default_rng(SEED + f).standard_normal((4200, f)), R)


@pytest.mark.parametrize("f", [64, 256, 7, 602])
def test_values_that_are_no_relation_are_skipped(world, f):
    R = 3
    rng = np.random.default_rng(SEED + 3 * f)
    rowStart, col_idx = csr_block(rng, 300, 300)
    vals = relations(rng, len(col_idx), R)
    bad = [R if b is None else b for b in NOT_RELATIONS]
    vals[::5] = np.resize(bad, len(vals[::5]))
    assert (~ro.valid(vals, R)).sum() >= 6
    check_kernels(rowStart, col_idx, vals, rng.standard_normal((300, f)), R)
    check_kernels(rowStart, col_idx, vals, rng.standard_normal((300, f)), R, (None, None), (None, None), 1)


def test_window_scale_and_relation_check(world):
    rng = np.random.default_rng(SEED + 7)
    n, f, R = 50, 5, 3
    counts = rng.integers(0, 4, (n, R)).astype(np.float64)
    A = rng.standard_normal((n, R * f))
    Ad, Cd = _dev_rows(A, R * f + 2, 0), _dev_rows(counts, R + 1, 0)
    assert lib().hnh_window_scale_f64(Ad.data_ptr(), R * f + 2, Cd.data_ptr(), R + 1, n, f, R, _st()) == 0
    torch.cuda.synchronize()
    c = counts.repeat(f, 1)
    want = np.divide(A, c, out=np.zeros_like(A), where=c != 0)
    assert np.array_equal(_host_rows(Ad, n, R * f, R * f + 2, 0), want)
    vals = torch.tensor([0.0, 2.0, 1.0, -1.0, 3.0, 0.5, math.nan, math.inf, -0.0, 2.0], dtype=torch.float64, device=DEV)
    bad = torch.full((1,), 10.0, dtype=torch.float64, device=DEV)
    assert lib().hnh_relation_check_f64(bad.data_ptr(), vals.data_ptr(), 10, R, _st()) == 0
    torch.cuda.synchronize()
    assert bad.item() == 15.0  # adds the 5 values that are no relation


# ---- the op at p = 1 ----------------------------------------------------------------------------------------------------
def op_case(alg_name, f, R, logM=7, npr=5):
    N = 1 << logM
    rows, cols, _ = orc.er_tuples(logM, npr, SEED + f)
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    rows, cols = np.append(rows, [3, 3, 3]), np.append(cols, [cols[0]] * 3)  # duplicates
    keep = rows != 9  # an empty row
    rows, cols = rows[keep], cols[keep]
    rels = relations(np.random.default_rng(SEED + 4), len(rows), R)
    rels[-3:] = [0, 1, 1]  # the duplicates under two relations
    S = D.SpmatLocal.from_tuples(N, N, rows, cols, rels)
    alg = D.Algorithm(alg_name, S, 8, 1)
    X = np.random.default_rng(SEED + 5).standard_normal((N, f))
    return N, rows, cols, rels, S, alg, X


@pytest.mark.parametrize("f", [8, 64, 13, 300])
@pytest.mark.parametrize("alg_name", ALGS)
def test_relational_aggregate_op(world, alg_name, f):
    R = 3
    N, rows, cols, rels, S, alg, X = op_case(alg_name, f, R)
    nA, nB = alg.like_A_matrix().shape[0], alg.like_B_matrix().shape[0]
    Xd, A = D.Dense.create(nB, f), D.Dense.create(nA, R * f, 7.0)
    Xh = np.zeros((nB, f))
    Xh[:N] = X
    Xd.from_host(Xh)
    alg.relational_aggregate(Xd, A, R)
    want = ro.relational_aggregate(rows, cols, rels, N, X, R)
    got = A.to_host()
    assert np.abs(got[:N] - want).max() <= 1e-13 * np.abs(want).max()
    assert not got[9].any() and not got[N:].any()  # the empty row and the padding
    dAh = np.zeros((nA, R * f))
    dAh[:N] = np.random.default_rng(SEED + 6).standard_normal((N, R * f))
    dA, dX = D.Dense.create(nA, R * f), D.Dense.create(nB, f, 3.0)
    dA.from_host(dAh)
    wdX = ro.relational_aggregate_backward(rows, cols, rels, dAh[:N], N, R)
    alg.relational_aggregate_backward(dA, dX, R)
    assert np.abs(dX.to_host()[:N] - wdX).max() <= 1e-13 * np.abs(wdX).max()
    first = dX.to_host()
    alg.relational_aggregate_backward(dA, dX, R, accumulate=True)
    assert np.abs(dX.to_host()[:N] - 2 * wdX).max() <= 1e-13 * np.abs(wdX).max()
    A2 = D.Dense.create(nA, R * f)
    alg.relational_aggregate(Xd, A2, R)
    dX2 = D.Dense.create(nB, f)
    alg.relational_aggregate_backward(dA, dX2, R)
    assert np.array_equal(A2.to_host(), got) and np.array_equal(dX2.to_host(), first)


def test_relational_aggregate_refusals(world):
    R = 3
    N, rows, cols, rels, S, alg, X = op_case("15d_fusion1", 8, R)
    nA, nB = alg.like_A_matrix().shape[0], alg.like_B_matrix().shape[0]
    Xd, A, dX = D.Dense.create(nB, 8), D.Dense.create(nA, R * 8), D.Dense.create(nB, 8)
    for args, msg in (((Xd, A, 0), "relation count must be positive"), ((Xd, D.Dense.create(nA, 8), R), "A-shaped"),
                      ((D.Dense.create(nB, 0), D.Dense.create(nA, 0), R), "width f must be positive"),
                      ((D.Dense.create(nB + 1, 8), A, R), "like_B_matrix"), ((Xd, Xd, 1), "another operand")):
        with pytest.raises(RuntimeError, match=msg):
            alg.relational_aggregate(*args)
    with pytest.raises(RuntimeError, match="A-shaped"):
        alg.relational_aggregate_backward(D.Dense.create(nA, 8), dX, R)
    with pytest.raises(RuntimeError, match="relation count"):
        alg.relational_aggregate_backward(A, dX, -1)
    with pytest.raises(RuntimeError, match="another operand"):
        alg.relational_aggregate_backward(Xd, Xd, 1)


# ---- the model ----------------------------------------------------------------------------------------------------------
def build(layers, aggr, R, logM=7, npr=5, alg_name="15d_fusion1", pattern=None, seed=SEED):
    N = 1 << logM
    if pattern is None:
        rows, cols, _ = orc.er_tuples(logM, npr, seed)
        rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
        rels = np.random.default_rng(seed + 2).integers(0, R, len(rows)).astype(np.float64)
    else:
        rows, cols, rels = pattern
    S = D.SpmatLocal.from_tuples(N, N, rows, cols, rels)
    alg = D.Algorithm(alg_name, S, layers[0][0], 1)
    net = D.RGCN(alg, layers, num_relations=R, aggr=aggr)
    rng = np.random.default_rng(seed + 1)
    params = ro.random_params(layers, R, rng)
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
    return dict(N=N, rows=rows, cols=cols, rels=rels, S=S, alg=alg, net=net, params=params, X=X, G=G, layers=layers, aggr=aggr, R=R)


def rel_err(got, ref):
    return np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-300)


def check_against_model(P):
    net, N, layers = P["net"], P["N"], P["layers"]
    net.forward()
    out, dX, dP = ro.forward_backward(P["rows"], P["cols"], P["rels"], N, layers, P["params"], P["X"], P["R"], P["aggr"],
                                      P["G"][:N])
    assert np.abs(out).max() > 0
    assert rel_err(net.buffer(len(layers))[:N], out) < 1e-10
    net.backward(P["G"])
    assert rel_err(net.input_grad()[:N], dX) < 1e-10
    for l, grads in enumerate(dP):
        for name, g in grads.items():
            got = net.param_grad(l, name)
            assert got.shape == g.shape, (l, name)
            assert rel_err(got, g) < 1e-10, (l, name, rel_err(got, g))


LAYER_SETS = {1: [(6, 4)], 2: [(6, 8), (8, 3)], 3: [(6, 8), (8, 5), (5, 4)]}


@pytest.mark.parametrize("R", [1, 4])
@pytest.mark.parametrize("aggr", ro.AGGREGATIONS)
@pytest.mark.parametrize("n_layers", [1, 2, 3])
def test_model_matches_oracle(world, n_layers, aggr, R):
    check_against_model(build(LAYER_SETS[n_layers], aggr, R))


def pattern_with_duplicates(R, N=128, nnz=500):
    rng = np.random.default_rng(SEED + 9)
    rows, cols = rng.integers(0, N, nnz), rng.integers(0, N, nnz)
    rows[rows % 7 == 0] = 1  # rows without entries and a hub row
    rows[:5], cols[:5] = 2, 11  # duplicates ...
    rels = rng.integers(0, R, nnz).astype(np.float64)
    rels[:5] = np.arange(5) % R  # ... under several relations
    return rows, cols, rels


@pytest.mark.parametrize("aggr", ro.AGGREGATIONS)
@pytest.mark.parametrize("alg_name", ALGS)
def test_model_on_every_algorithm_with_duplicates_and_empty_rows(world, alg_name, aggr):
    check_against_model(build([(6, 64), (64, 3)], aggr, 4, alg_name=alg_name, pattern=pattern_with_duplicates(4)))


@pytest.mark.parametrize("aggr", ro.AGGREGATIONS)
def test_wide_input_layer(world, aggr):
    check_against_model(build([(602, 16), (16, 4)], aggr, 4, logM=8))


def test_one_relation_matches_graph_sage_mean(world):
    layers = [(6, 8), (8, 3)]
    P = build(layers, "mean", 1)
    N = P["N"]
    S2 = D.SpmatLocal.from_tuples(N, N, P["rows"], P["cols"], np.ones(len(P["rows"])))
    alg2 = D.Algorithm("15d_fusion1", S2, 6, 1)
    sage = D.GraphSAGE(alg2, layers, aggr="mean")
    for l, Pl in enumerate(P["params"]):
        sage.set_param(l, "neigh", Pl["weight"])
        sage.set_param(l, "neigh_bias", Pl["bias"])
        sage.set_param(l, "root", Pl["root"])
    Xl = np.zeros(sage.buffer_shape(0))
    Xl[:N] = P["X"]
    sage.set_input(Xl)
    net = P["net"]
    for m in (net, sage):
        m.forward()
        m.backward(P["G"])
    assert rel_err(net.buffer(2)[:N], sage.buffer(2)[:N]) < 1e-12
    assert rel_err(net.input_grad()[:N], sage.input_grad()[:N]) < 1e-12
    for l in range(2):
        for mine, theirs in (("weight", "neigh"), ("bias", "neigh_bias"), ("root", "root")):
            assert rel_err(net.param_grad(l, mine), sage.param_grad(l, theirs)) < 1e-12, (l, mine)


def test_backward_repeats_bit_identical_and_needs_a_forward(world):
    P = build(LAYER_SETS[2], "mean", 4)
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


def test_rgcn_model_refusals(world):
    P = build(LAYER_SETS[1], "sum", 3)
    alg, net = P["alg"], P["net"]
    out = C.c_void_p()
    flat = (C.c_int * 2)(6, 4)
    assert lib().hnhd_rgcn_create(alg.h, 1, flat, 3, b"max", C.byref(out)) == -1
    assert b"unknown aggregation" in lib().hnh_last_error_string()
    assert lib().hnhd_rgcn_create(alg.h, 1, flat, 0, b"sum", C.byref(out)) == -1
    assert lib().hnhd_rgcn_create(alg.h, 2, (C.c_int * 4)(6, 4, 5, 3), 3, b"sum", C.byref(out)) == -1
    assert b"does not take the width" in lib().hnh_last_error_string()
    for name in (b"query", b"neigh"):
        r, c = C.c_int64(), C.c_int64()
        assert lib().hnhd_model_param_shape(net.h, 0, name, C.byref(r), C.byref(c)) == -1
        assert b"no parameter" in lib().hnh_last_error_string()
    with pytest.raises(RuntimeError, match="no such layer"):
        net.param(1, "root")
    assert net.param_shape(0, "weight") == (18, 4) and net.param_shape(0, "bias") == (4,) and net.param_shape(0, "root") == (6, 4)
    # a stored value that is no relation is refused at construction
    rows, cols, rels = P["rows"], P["cols"], P["rels"].copy()
    rels[5] = 3.0
    S = D.SpmatLocal.from_tuples(P["N"], P["N"], rows, cols, rels)
    alg2 = D.Algorithm("15d_fusion1", S, 6, 1)
    with pytest.raises(RuntimeError, match="not integers in"):
        D.RGCN(alg2, LAYER_SETS[1], num_relations=3)
    D.RGCN(alg2, LAYER_SETS[1], num_relations=4)  # the same values are relations when R = 4


# ---- training -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("aggr", ro.AGGREGATIONS)
def test_train_step_matches_torch_adamw(world, aggr):
    P = build([(6, 8), (8, 3)], aggr, 3)
    N = P["N"]
    rng = np.random.default_rng(SEED + 11)
    labels = rng.integers(0, 3, N)
    labels[rng.random(N) < 0.3] = -1
    lab = np.full(P["net"].buffer_shape(2)[0], -1)
    lab[:N] = labels
    L = D.NodeLabels(P["net"], lab, 3)
    opt = D.AdamW(lr=1e-2, max_grad_norm=0.5)
    got = [P["net"].train_step(L, opt) for _ in range(5)]
    res, trained = ro.train(P["rows"], P["cols"], P["rels"], N, P["layers"], P["params"], P["X"], 3, aggr, labels, 5, lr=1e-2,
                            max_grad_norm=0.5)
    for g, w in zip(got, res):
        assert abs(g.loss - w[0]) <= 1e-10 * abs(w[0]) and abs(g.grad_norm - w[3]) <= 1e-10 * abs(w[3])
        assert (g.correct, g.labelled) == (w[1], w[2])
    for l, Pt in enumerate(trained):
        for k, v in Pt.items():
            assert np.abs(P["net"].param(l, k) - v).max() <= 1e-9 * max(np.abs(v).max(), 1.0), (l, k)


@pytest.mark.parametrize("aggr", ro.AGGREGATIONS)
def test_link_train_step_matches_torch_adamw(world, aggr):
    P = build([(6, 8), (8, 4)], aggr, 3)
    N = P["N"]
    rng = np.random.default_rng(SEED + 12)
    tr, tc = rng.integers(0, N, 4 * N), rng.integers(0, N, 4 * N)
    y = rng.choice([0.0, 1.0], 4 * N)
    algT = D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, tr, tc, y), 6, 1)
    t = D.LinkTargets(P["net"], algT)
    opt = D.AdamW(lr=1e-2)
    got = [P["net"].link_train_step(t, opt) for _ in range(4)]
    res, trained = ro.train_link(P["rows"], P["cols"], P["rels"], N, P["layers"], P["params"], P["X"], 3, aggr, (tr, tc, y), 4,
                                 lr=1e-2)
    for g, w in zip(got, res):
        assert abs(g.loss - w[0]) <= 1e-10 * abs(w[0]) and abs(g.grad_norm - w[3]) <= 1e-10 * abs(w[3])
        assert g.labelled == w[2] and abs(g.correct - w[1]) <= 1
    for l, Pt in enumerate(trained):
        for k, v in Pt.items():
            assert np.abs(P["net"].param(l, k) - v).max() <= 1e-9 * max(np.abs(v).max(), 1.0), (l, k)
    loss, correct, count, scores = P["net"].link_evaluate(t)
    H = P["net"].buffer(2)[:N]
    er, ec = algT.entry_coordinates("A")
    want = (H[er] * H[ec]).sum(1)
    assert count == 4 * N and np.abs(scores - want).max() <= 1e-12 * np.abs(want).max()
