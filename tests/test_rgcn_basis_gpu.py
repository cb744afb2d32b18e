"""R-GCN with basis decomposition on the GPU on one rank.  The kernels hnh_basis_aggregate_f64 / _grad_f64 (with the
per-entry products) against numpy at every table width, at odd widths and past 256 (column windows), at B = 1, 3, 8
and 30 (more bases than the registers hold: chunked) and R = 1, 3 and 64 with one relation without entries, with the
mean's scale and without one, at odd leading dimensions and misaligned rows with NaN guard cells untouched, with empty
rows, hub rows and duplicates under different relations, values that are no relation (skipped, P = 0), more rows than
one resident wave, the skewed graph, and bit-identical repeats.  The op Distributed_Sparse::basisAggregate /
basisAggregateBackward at p = 1 under every algorithm; the model's forward, backward and every gradient against
tests/rgcn_basis_oracle.py; the basis model with B = R and comp = I against the model without bases; train_step and
link_train_step against a torch AdamW loop; refusals.  Multi-rank cases are in tests/test_rgcn_basis_multirank_gpu.py."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from distributed_sddmm_b200 import driver as D
from distributed_sddmm_b200 import lib
from oracle import hnh_oracle as orc
from tests import rgcn_basis_oracle as bo
from tests import rgcn_oracle as ro
from tests.skewed_graph import skewed_tuples
from tests.test_link_prediction_gpu import csr_block
from tests.test_rgcn_gpu import NOT_RELATIONS, _dev_rows, _host_rows, _st, relations, rel_err

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
SEED = 0xC0FFEE + 263
ALGS = ["15d_fusion1", "15d_fusion2", "15d_sparse", "25d_dense_replicate", "25d_sparse_replicate"]


@pytest.fixture(scope="module")
def world():
    D.world_init("self")
    yield
    D.world_finalize()


# ---- the kernels --------------------------------------------------------------------------------------------------------
def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def run_aggregate(rowStart, col_idx, vals, X, H0, comp, scale, ld=(None, None, None), offset=0):
    """ld = (ldx, lds, ldh)."""
    n, f, R, B = len(rowStart) - 1, X.shape[1], comp.shape[0], comp.shape[1]
    ldx, lds, ldh = ld[0] or f, ld[1] or R, ld[2] or B * f
    xb, hb = _dev_rows(X, ldx, offset), _dev_rows(H0, ldh, offset)
    sb = _dev_rows(scale, lds, offset) if scale is not None else None
    rs, ci, v, cp = (_dev(a) for a in (rowStart, col_idx, vals, comp))
    p = lambda b: b.data_ptr() + 8 * offset  # noqa: E731
    rc = lib().hnh_basis_aggregate_f64(rs.data_ptr(), ci.data_ptr(), v.data_ptr(), n, len(col_idx), p(xb), ldx, f,
                                       p(sb) if sb is not None else None, lds, cp.data_ptr(), R, B, p(hb), ldh, _st())
    assert rc == 0, lib().hnh_last_error_string()
    torch.cuda.synchronize()
    if sb is not None:
        assert np.array_equal(_host_rows(sb, n, R, lds, offset), scale)
    return _host_rows(hb, n, B * f, ldh, offset)


def run_grad(rowStart, col_idx, vals, dH, X, dX0, comp, scale, ld=(None, None, None, None), offset=0, with_p=True):
    """ld = (lddh, lds, ldx, lddx); returns (dX, P (B x nnz) or None)."""
    m, f, R, B = len(rowStart) - 1, dX0.shape[1], comp.shape[0], comp.shape[1]
    nnz, n = len(col_idx), dH.shape[0]
    lddh, lds, ldx, lddx = ld[0] or B * f, ld[1] or R, ld[2] or f, ld[3] or f
    ldp = nnz + 3
    hb, xb, dxb = _dev_rows(dH, lddh, offset), _dev_rows(X, ldx, offset), _dev_rows(dX0, lddx, offset)
    sb = _dev_rows(scale, lds, offset) if scale is not None else None
    pb = _dev_rows(np.zeros((B, nnz)), ldp, offset) if with_p else None
    if with_p:
        pb[offset:offset + B * ldp].view(B, ldp)[:, :nnz] = math.nan  # every product is written
    rs, ci, v, cp = (_dev(a) for a in (rowStart, col_idx, vals, comp))
    p = lambda b: b.data_ptr() + 8 * offset if b is not None else None  # noqa: E731
    rc = lib().hnh_basis_aggregate_grad_f64(rs.data_ptr(), ci.data_ptr(), v.data_ptr(), m, nnz, p(hb), lddh, p(sb), lds,
                                            cp.data_ptr(), R, B, p(xb), ldx, f, p(dxb), lddx, p(pb), ldp, _st())
    assert rc == 0, lib().hnh_last_error_string()
    torch.cuda.synchronize()
    assert np.array_equal(_host_rows(hb, n, B * f, lddh, offset), dH) and np.array_equal(_host_rows(xb, m, f, ldx, offset), X)
    P = _host_rows(pb, B, nnz, ldp, offset) if with_p else None
    return _host_rows(dxb, m, f, lddx, offset), P


def check_kernels(rowStart, col_idx, vals, X, R, B, mean=True, ld_agg=(None, None, None), ld_grad=(None, None, None, None),
                  offset=0):
    """The aggregate into a pre-filled H and the grad into a pre-filled dX with the products, against numpy; repeats
    bit-identical."""
    n, m, f = len(rowStart) - 1, X.shape[0], X.shape[1]
    rows = np.repeat(np.arange(n), np.diff(rowStart))
    rng = np.random.default_rng(f + R + 100 * B)
    comp = rng.standard_normal((R, B))
    scale = bo.mean_scale(rows, vals, n, R) if mean else None
    H0 = rng.standard_normal((n, B * f))
    H = run_aggregate(rowStart, col_idx, vals, X, H0, comp, scale, ld_agg, offset)
    want = H0 + bo.basis_aggregate(rows, col_idx, vals, n, X, R, comp, scale)
    assert np.abs(H - want).max() <= 1e-12 * max(np.abs(want).max(), 1.0)
    assert np.array_equal(H[np.diff(rowStart) == 0], H0[np.diff(rowStart) == 0])  # rows without entries are not written
    assert np.array_equal(run_aggregate(rowStart, col_idx, vals, X, H0, comp, scale, ld_agg, offset), H)
    # grad on the transposed block (the rows of X are its stored rows, dH and scale are gathered)
    order = np.lexsort((rows, col_idx))
    tr, tc, tv = col_idx[order], rows[order], vals[order]
    tStart = np.searchsorted(tr, np.arange(m + 1)).astype(np.int64)
    dH = rng.standard_normal((n, B * f))
    Xs = rng.standard_normal((m, f))  # the stored rows' X, read for the products
    dX0 = rng.standard_normal((m, f))
    dX, P = run_grad(tStart, tc, tv, dH, Xs, dX0, comp, scale, ld_grad, offset)
    wdX, _ = bo.basis_aggregate_backward(rows, col_idx, vals, dH, Xs, m, R, comp, scale)
    assert np.abs(dX - (dX0 + wdX)).max() <= 1e-12 * max(np.abs(wdX).max(), 1.0)
    wP = bo.products(tc, tr, tv, dH, Xs, R, B, scale)
    assert np.abs(P - wP).max() <= 1e-12 * max(np.abs(wP).max(), 1.0)
    assert not P[:, ~ro.valid(tv, R)].any()  # entries that are no relation: P = 0
    dX2, P2 = run_grad(tStart, tc, tv, dH, Xs, dX0, comp, scale, ld_grad, offset)
    assert np.array_equal(dX2, dX) and np.array_equal(P2, P)  # bit-identical repeats
    dX3, _ = run_grad(tStart, tc, tv, dH, Xs, dX0, comp, scale, ld_grad, offset, with_p=False)
    assert np.array_equal(dX3, dX)  # the products do not change dX


WIDTHS = [1, 3, 4, 8, 16, 32, 64, 100, 128, 256, 257, 602]


@pytest.mark.parametrize("R,B", [(1, 1), (3, 3), (64, 8), (3, 30)])
@pytest.mark.parametrize("f", WIDTHS)
def test_basis_kernels_match_numpy(world, f, R, B):
    rng = np.random.default_rng(SEED + f + 1000 * R + 7 * B)
    rowStart, col_idx = csr_block(rng, 300, 300)  # empty rows, duplicates, a hub row of 150 entries
    check_kernels(rowStart, col_idx, relations(rng, len(col_idx), R), rng.standard_normal((300, f)), R, B)


@pytest.mark.parametrize("B", [4, 30])
@pytest.mark.parametrize("f", [4, 16, 128, 7, 602])
def test_basis_kernels_without_scale(world, f, B):
    rng = np.random.default_rng(SEED + 3 * f + B)
    rowStart, col_idx = csr_block(rng, 300, 300)
    check_kernels(rowStart, col_idx, relations(rng, len(col_idx), 5), rng.standard_normal((300, f)), 5, B, mean=False)


@pytest.mark.parametrize("f", [4, 64, 256, 5, 602])
def test_basis_kernels_odd_ld_and_misaligned_rows(world, f):
    rng = np.random.default_rng(SEED + 2 * f)
    R, B = 3, 4
    rowStart, col_idx = csr_block(rng, 200, 200)
    vals = relations(rng, len(col_idx), R)
    X = rng.standard_normal((200, f))
    for ld_agg, ld_grad, offset in (((f + 1, R + 1, None), (B * f + 1, R + 1, None, None), 0),
                                    ((None, None, B * f + 1), (None, None, f + 1, f + 1), 0),
                                    ((None, None, None), (None, None, None, None), 1)):
        check_kernels(rowStart, col_idx, vals, X, R, B, True, ld_agg, ld_grad, offset)


@pytest.mark.parametrize("f,n", [(4, 200000), (64, 30000), (256, 12000), (5, 40000)])
def test_basis_kernels_past_one_wave(world, f, n):
    rng = np.random.default_rng(SEED + n)
    rowStart, col_idx = csr_block(rng, n, n, per_row=3)
    check_kernels(rowStart, col_idx, relations(rng, len(col_idx), 8), rng.standard_normal((n, f)), 8, 4)


@pytest.mark.parametrize("f,B", [(64, 4), (7, 3), (16, 30)])
def test_basis_kernels_on_the_skewed_graph(world, f, B):
    R = 5
    rows, cols = skewed_tuples(4200, 4200, SEED)
    rows, cols = rows.astype(np.int64), cols.astype(np.int64)
    vals = ro.hashed_relations(rows, cols, 4200, R)
    order = np.lexsort((cols, rows))
    rows, cols, vals = rows[order], cols[order], vals[order]
    rowStart = np.searchsorted(rows, np.arange(4201)).astype(np.int64)
    check_kernels(rowStart, cols, vals, np.random.default_rng(SEED + f).standard_normal((4200, f)), R, B)


@pytest.mark.parametrize("f", [64, 256, 7, 602])
def test_values_that_are_no_relation_are_skipped(world, f):
    R = 3
    rng = np.random.default_rng(SEED + 5 * f)
    rowStart, col_idx = csr_block(rng, 300, 300)
    vals = relations(rng, len(col_idx), R)
    vals[::5] = np.resize([R if b is None else b for b in NOT_RELATIONS], len(vals[::5]))
    assert (~ro.valid(vals, R)).sum() >= 6
    X = rng.standard_normal((300, f))
    check_kernels(rowStart, col_idx, vals, X, R, 4)
    check_kernels(rowStart, col_idx, vals, X, R, 4, False, (None, None, None), (None, None, None, None), 1)


def test_relation_keys(world):
    vals = torch.tensor([0.0, 2.0, 1.0, -1.0, 3.0, 0.5, math.nan, math.inf, -0.0, 2.0], dtype=torch.float64, device=DEV)
    keys = torch.full((11,), -7, dtype=torch.int32, device=DEV)
    assert lib().hnh_relation_keys(keys.data_ptr(), vals.data_ptr(), 10, 3, _st()) == 0
    torch.cuda.synchronize()
    assert keys.tolist() == [0, 2, 1, 3, 3, 3, 3, 3, 0, 2, -7]


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


def _padded(M, rows):
    out = np.zeros((rows,) + M.shape[1:])
    out[:len(M)] = M
    return out


@pytest.mark.parametrize("mean", [False, True])
@pytest.mark.parametrize("f", [8, 64, 13, 300])
@pytest.mark.parametrize("alg_name", ALGS)
def test_basis_aggregate_op(world, alg_name, f, mean):
    R, B = 3, 2
    N, rows, cols, rels, S, alg, X = op_case(alg_name, f, R)
    nA, nB = alg.like_A_matrix().shape[0], alg.like_B_matrix().shape[0]
    comp = np.random.default_rng(SEED + 7).standard_normal((R, B))
    sc = bo.mean_scale(rows, rels, N, R) if mean else None
    scale = None
    if mean:
        scale = D.Dense.create(nA, R)
        scale.from_host(_padded(sc, nA))
    Xd, H = D.Dense.create(nB, f), D.Dense.create(nA, B * f, 7.0)
    Xd.from_host(_padded(X, nB))
    alg.basis_aggregate(Xd, H, comp, R, scale)
    want = bo.basis_aggregate(rows, cols, rels, N, X, R, comp, sc)
    got = H.to_host()
    assert np.abs(got[:N] - want).max() <= 1e-12 * np.abs(want).max()
    assert not got[9].any() and not got[N:].any()  # the empty row and the padding
    dHh = _padded(np.random.default_rng(SEED + 6).standard_normal((N, B * f)), nA)
    dH, dX = D.Dense.create(nA, B * f), D.Dense.create(nB, f, 3.0)
    dH.from_host(dHh)
    wdX, wdcomp = bo.basis_aggregate_backward(rows, cols, rels, dHh[:N], X, N, R, comp, sc)
    dcomp = alg.basis_aggregate_backward(dH, Xd, dX, comp, R, scale)
    assert np.abs(dX.to_host()[:N] - wdX).max() <= 1e-12 * np.abs(wdX).max()
    assert dcomp.shape == (R, B) and np.abs(dcomp - wdcomp).max() <= 1e-12 * np.abs(wdcomp).max()
    first = dX.to_host()
    dcomp2 = alg.basis_aggregate_backward(dH, Xd, dX, comp, R, scale, accumulate=True)
    assert np.abs(dX.to_host()[:N] - 2 * wdX).max() <= 1e-12 * np.abs(wdX).max()
    H2, dX2 = D.Dense.create(nA, B * f), D.Dense.create(nB, f)
    alg.basis_aggregate(Xd, H2, comp, R, scale)
    dcomp3 = alg.basis_aggregate_backward(dH, Xd, dX2, comp, R, scale)
    assert np.array_equal(H2.to_host(), got) and np.array_equal(dX2.to_host(), first)
    assert np.array_equal(dcomp2, dcomp) and np.array_equal(dcomp3, dcomp)


def test_basis_aggregate_refusals(world):
    R, B, f = 3, 2, 8
    N, rows, cols, rels, S, alg, X = op_case("15d_fusion1", f, R)
    nA, nB = alg.like_A_matrix().shape[0], alg.like_B_matrix().shape[0]
    comp = D.Dense.create(R, B)
    Xd, H, dX = D.Dense.create(nB, f), D.Dense.create(nA, B * f), D.Dense.create(nB, f)
    for args, msg in (((Xd, H, comp, 0), "relation count must be positive"), ((Xd, H, np.ones((R + 1, B)), R), "comp is"),
                      ((Xd, D.Dense.create(nA, f), comp, R), "A-shaped"), ((D.Dense.create(nB + 1, f), H, comp, R), "like_B_matrix"),
                      ((Xd, H, comp, R, D.Dense.create(nA, R + 1)), "scale is"), ((Xd, Xd, np.ones((R, 1)), R), "another operand"),
                      ((Xd, H, comp, R, H), "scale is"), ((Xd, comp, np.ones((R, 1)), R), "A-shaped")):
        with pytest.raises(RuntimeError, match=msg):
            alg.basis_aggregate(*args)
    with pytest.raises(RuntimeError, match="another operand"):
        alg.basis_aggregate_backward(H, Xd, Xd, comp, R)
    with pytest.raises(RuntimeError, match="A-shaped"):
        alg.basis_aggregate_backward(D.Dense.create(nA, f), Xd, dX, comp, R)
    with pytest.raises(RuntimeError, match="B-shaped"):
        alg.basis_aggregate_backward(H, Xd, D.Dense.create(nB, f + 1), comp, R)
    with pytest.raises(RuntimeError, match="relation count"):
        alg.basis_aggregate_backward(H, Xd, dX, comp, -1)
    with pytest.raises(RuntimeError, match="comp is"):
        alg.basis_aggregate_backward(H, Xd, dX, np.ones((R - 1, B)), R)
    with pytest.raises(RuntimeError, match="scale is"):
        alg.basis_aggregate_backward(H, Xd, dX, comp, R, dX)


# ---- the model ----------------------------------------------------------------------------------------------------------
def build(layers, aggr, R, B, logM=7, npr=5, alg_name="15d_fusion1", pattern=None, seed=SEED, params=None):
    N = 1 << logM
    if pattern is None:
        rows, cols, _ = orc.er_tuples(logM, npr, seed)
        rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
        rels = np.random.default_rng(seed + 2).integers(0, R, len(rows)).astype(np.float64)
    else:
        rows, cols, rels = pattern
    S = D.SpmatLocal.from_tuples(N, N, rows, cols, rels)
    alg = D.Algorithm(alg_name, S, layers[0][0], 1)
    net = D.RGCN(alg, layers, num_relations=R, aggr=aggr, num_bases=B)
    rng = np.random.default_rng(seed + 1)
    params = params or bo.random_params(layers, R, B, rng)
    for l, P in enumerate(params):
        for name, v in P.items():
            net.set_param(l, name, v)
    X = rng.uniform(-1, 1, (N, layers[0][0]))
    net.set_input(_padded(X, net.buffer_shape(0)[0]))
    shape = net.buffer_shape(len(layers))
    G = np.zeros(shape)
    G[:N] = rng.uniform(-1, 1, (N, shape[1]))
    return dict(N=N, rows=rows, cols=cols, rels=rels, S=S, alg=alg, net=net, params=params, X=X, G=G, layers=layers, aggr=aggr,
                R=R, B=B)


def check_against_model(P):
    net, N, layers = P["net"], P["N"], P["layers"]
    net.forward()
    out, dX, dP = bo.forward_backward(P["rows"], P["cols"], P["rels"], N, layers, P["params"], P["X"], P["R"], P["B"], P["aggr"],
                                      P["G"][:N])
    assert np.abs(out).max() > 0
    assert rel_err(net.buffer(len(layers))[:N], out) < 1e-10
    net.backward(P["G"])
    assert rel_err(net.input_grad()[:N], dX) < 1e-10
    for l, grads in enumerate(dP):
        assert sorted(grads) == sorted(net.param_names())
        for name, g in grads.items():
            got = net.param_grad(l, name)
            assert got.shape == g.shape, (l, name)
            assert rel_err(got, g) < 1e-10, (l, name, rel_err(got, g))


LAYER_SETS = {1: [(6, 4)], 2: [(6, 8), (8, 3)], 3: [(6, 8), (8, 5), (5, 4)]}


@pytest.mark.parametrize("R,B", [(1, 1), (5, 2), (4, 30)])
@pytest.mark.parametrize("aggr", bo.AGGREGATIONS)
@pytest.mark.parametrize("n_layers", [1, 2, 3])
def test_model_matches_oracle(world, n_layers, aggr, R, B):
    check_against_model(build(LAYER_SETS[n_layers], aggr, R, B))


def pattern_with_duplicates(R, N=128, nnz=500):
    rng = np.random.default_rng(SEED + 9)
    rows, cols = rng.integers(0, N, nnz), rng.integers(0, N, nnz)
    rows[rows % 7 == 0] = 1  # rows without entries and a hub row
    rows[:5], cols[:5] = 2, 11  # duplicates ...
    rels = rng.integers(0, R, nnz).astype(np.float64)
    rels[:5] = np.arange(5) % R  # ... under several relations
    return rows, cols, rels


@pytest.mark.parametrize("aggr", bo.AGGREGATIONS)
@pytest.mark.parametrize("alg_name", ALGS)
def test_model_on_every_algorithm_with_duplicates_and_empty_rows(world, alg_name, aggr):
    check_against_model(build([(6, 64), (64, 3)], aggr, 6, 3, alg_name=alg_name, pattern=pattern_with_duplicates(6)))


@pytest.mark.parametrize("aggr", bo.AGGREGATIONS)
def test_wide_input_layer(world, aggr):
    check_against_model(build([(602, 16), (16, 4)], aggr, 8, 3, logM=8))


@pytest.mark.parametrize("aggr", bo.AGGREGATIONS)
def test_identity_bases_match_the_model_without_bases(world, aggr):
    """B = R and comp = I: the forward and every shared gradient of the two paths agree to 1e-12."""
    layers, R = [(6, 8), (8, 3)], 4
    params = bo.random_params(layers, R, R, np.random.default_rng(SEED + 13))
    for Pl in params:
        Pl["comp"] = np.eye(R)
    P = build(layers, aggr, R, R, params=params)
    net, N = P["net"], P["N"]
    alg2 = D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, P["rows"], P["cols"], P["rels"]), 6, 1)
    plain = D.RGCN(alg2, layers, num_relations=R, aggr=aggr)
    for l, Pl in enumerate(params):
        for k in ro.PARAMS:
            plain.set_param(l, k, Pl[k])
    plain.set_input(_padded(P["X"], plain.buffer_shape(0)[0]))
    for m in (net, plain):
        m.forward()
        m.backward(P["G"])
    assert rel_err(net.buffer(2)[:N], plain.buffer(2)[:N]) < 1e-12
    assert rel_err(net.input_grad()[:N], plain.input_grad()[:N]) < 1e-12
    for l in range(2):
        for k in ro.PARAMS:
            assert rel_err(net.param_grad(l, k), plain.param_grad(l, k)) < 1e-12, (l, k)


def test_backward_repeats_bit_identical_and_needs_a_forward(world):
    P = build(LAYER_SETS[2], "mean", 4, 2)
    net = P["net"]
    net.forward()
    net.backward(P["G"])
    first = [net.param_grad(l, n) for l in range(2) for n in net.param_names()] + [net.input_grad()]
    net.forward()
    net.backward(P["G"])
    again = [net.param_grad(l, n) for l in range(2) for n in net.param_names()] + [net.input_grad()]
    assert all(np.array_equal(a, b) for a, b in zip(first, again))
    net.set_param(0, "comp", P["params"][0]["comp"])
    with pytest.raises(RuntimeError, match="no forward pass"):
        net.backward(P["G"])


def test_model_refusals(world):
    P = build(LAYER_SETS[1], "sum", 3, 2)
    alg, net = P["alg"], P["net"]
    out = C.c_void_p()
    flat = (C.c_int * 2)(6, 4)
    assert lib().hnhd_rgcn_create_bases(alg.h, 1, flat, 3, 0, b"sum", C.byref(out)) == -1
    assert b"basis count" in lib().hnh_last_error_string()
    assert lib().hnhd_rgcn_create_bases(alg.h, 1, flat, 3, 2, b"max", C.byref(out)) == -1
    for name in (b"query", b"neigh", b"basis"):
        r, c = C.c_int64(), C.c_int64()
        assert lib().hnhd_rgcn_param_shape(net.h, 0, name, C.byref(r), C.byref(c)) == -1
        assert b"no parameter" in lib().hnh_last_error_string()
    assert net.param_names() == ["weight", "comp", "bias", "root"]
    assert net.param_shape(0, "weight") == (12, 4) and net.param_shape(0, "comp") == (3, 2)
    assert net.param_shape(0, "bias") == (4,) and net.param_shape(0, "root") == (6, 4)
    with pytest.raises(ValueError, match="is \\(3, 2\\)"):
        net.set_param(0, "comp", np.zeros((2, 3)))
    # a stored value that is no relation is refused at construction
    rels = P["rels"].copy()
    rels[5] = 3.0
    alg2 = D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(P["N"], P["N"], P["rows"], P["cols"], rels), 6, 1)
    with pytest.raises(RuntimeError, match="not integers in"):
        D.RGCN(alg2, LAYER_SETS[1], num_relations=3, num_bases=2)
    plain = D.RGCN(alg2, LAYER_SETS[1], num_relations=4)
    with pytest.raises(ValueError, match="no parameter"):
        plain.param_shape(0, "comp")
    r, c = C.c_int64(), C.c_int64()
    assert lib().hnhd_rgcn_param_shape(plain.h, 0, b"comp", C.byref(r), C.byref(c)) == -1


# ---- training -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("aggr", bo.AGGREGATIONS)
def test_train_step_matches_torch_adamw(world, aggr):
    R, B = 5, 2
    P = build([(6, 8), (8, 3)], aggr, R, B)
    N = P["N"]
    rng = np.random.default_rng(SEED + 11)
    labels = rng.integers(0, 3, N)
    labels[rng.random(N) < 0.3] = -1
    lab = np.full(P["net"].buffer_shape(2)[0], -1)
    lab[:N] = labels
    L = D.NodeLabels(P["net"], lab, 3)
    opt = D.AdamW(lr=1e-2, max_grad_norm=0.5)
    got = [P["net"].train_step(L, opt) for _ in range(5)]
    res, trained = bo.train(P["rows"], P["cols"], P["rels"], N, P["layers"], P["params"], P["X"], R, B, aggr, labels, 5, lr=1e-2,
                            max_grad_norm=0.5)
    for g, w in zip(got, res):
        assert abs(g.loss - w[0]) <= 1e-10 * abs(w[0]) and abs(g.grad_norm - w[3]) <= 1e-10 * abs(w[3])
        assert (g.correct, g.labelled) == (w[1], w[2])
    for l, Pt in enumerate(trained):
        for k, v in Pt.items():
            assert np.abs(P["net"].param(l, k) - v).max() <= 1e-9 * max(np.abs(v).max(), 1.0), (l, k)


@pytest.mark.parametrize("aggr", bo.AGGREGATIONS)
def test_link_train_step_matches_torch_adamw(world, aggr):
    R, B = 5, 3
    P = build([(6, 8), (8, 4)], aggr, R, B)
    N = P["N"]
    rng = np.random.default_rng(SEED + 12)
    tr, tc = rng.integers(0, N, 4 * N), rng.integers(0, N, 4 * N)
    y = rng.choice([0.0, 1.0], 4 * N)
    algT = D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, tr, tc, y), 6, 1)
    t = D.LinkTargets(P["net"], algT)
    opt = D.AdamW(lr=1e-2)
    got = [P["net"].link_train_step(t, opt) for _ in range(4)]
    res, trained = bo.train_link(P["rows"], P["cols"], P["rels"], N, P["layers"], P["params"], P["X"], R, B, aggr, (tr, tc, y), 4,
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
