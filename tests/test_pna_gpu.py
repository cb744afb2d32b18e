"""PNA and multi-statistic aggregation on the GPU on one rank.  The kernels hnh_multi_aggregate_step_f64 / _grad_f64
against numpy for every subset of {moments, max, min} at every table width, at odd widths and past 256 (column windows),
on normal, ReLU'd and integer inputs (ties, with -0.0 and +0.0), at odd leading dimensions and misaligned rows, past one
resident wave, on the skewed graph's hub rows, with the state carried across two blocks, and bit-identical repeats.  The
op Distributed_Sparse::multiAggregate / multiAggregateBackward at p = 1 under every algorithm; the model's forward,
input gradient and every parameter gradient against tests/pna_oracle.py's literal per-edge PNAConv; train_step,
link_train_step and graph_train_step against a torch AdamW loop; a learning check; refusals."""
import ctypes as C
import itertools

import numpy as np
import pytest
import torch

from distributed_sddmm_b200 import driver as D
from distributed_sddmm_b200 import lib
from oracle import hnh_oracle as orc
from tests import graph_readout_oracle as gro
from tests import pna_oracle as po
from tests.skewed_graph import skewed_tuples
from tests.test_graph_sage_gpu import _dev_rows, _host_rows, _st, inputs
from tests.test_link_prediction_gpu import csr_block

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
SEED = 0xC0FFEE + 313
ALGS = ["15d_fusion1", "15d_fusion2", "15d_sparse", "25d_dense_replicate", "25d_sparse_replicate"]
WIDTHS = [1, 3, 4, 8, 16, 32, 64, 100, 128, 256, 257, 602]
SUBSETS = [w for n in (1, 2, 3) for w in itertools.combinations(po.STATS, n)]


@pytest.fixture(scope="module")
def world():
    D.world_init("self")
    yield
    D.world_finalize()


def flags(which):
    return sum(D.Algorithm.MULTI_STATISTICS[w] for w in which)


# ---- the kernels --------------------------------------------------------------------------------------------------------
def initial_state(n, f, which):
    """(0, 0, -inf, 0, +inf, 0): the state before the first block."""
    parts = ([np.zeros((n, f))] * 2 if "moments" in which else []) + \
        ([np.full((n, f), -np.inf), np.zeros((n, f))] if "max" in which else []) + \
        ([np.full((n, f), np.inf), np.zeros((n, f))] if "min" in which else [])
    return np.hstack(parts)


def run_step(rowStart, col_idx, X, A0, which, ld=(None, None), offset=0):
    n, f, w = len(rowStart) - 1, X.shape[1], A0.shape[1]
    ldx, lda = ld[0] or f, ld[1] or w
    xb, ab = _dev_rows(X, ldx, offset), _dev_rows(A0, lda, offset)
    rs, ci = torch.from_numpy(rowStart).to(DEV), torch.from_numpy(col_idx).to(DEV)
    p = lambda b: b.data_ptr() + 8 * offset  # noqa: E731
    rc = lib().hnh_multi_aggregate_step_f64(rs.data_ptr(), ci.data_ptr(), n, len(col_idx), p(xb), ldx, f, flags(which), p(ab), lda,
                                            _st())
    assert rc == 0, lib().hnh_last_error_string()
    torch.cuda.synchronize()
    return _host_rows(ab, n, w, lda, offset)


def run_grad(rowStart, col_idx, X, Dm, dX0, which, ld=(None, None, None), offset=0):
    n, f, w = len(rowStart) - 1, X.shape[1], Dm.shape[1]
    ldx, ldd, lddx = ld[0] or f, ld[1] or w, ld[2] or f
    xb, db, ob = _dev_rows(X, ldx, offset), _dev_rows(Dm, ldd, offset), _dev_rows(dX0, lddx, offset)
    rs, ci = torch.from_numpy(rowStart).to(DEV), torch.from_numpy(col_idx).to(DEV)
    p = lambda b: b.data_ptr() + 8 * offset  # noqa: E731
    rc = lib().hnh_multi_aggregate_grad_f64(rs.data_ptr(), ci.data_ptr(), n, len(col_idx), p(xb), ldx, p(db), ldd, f, flags(which),
                                            p(ob), lddx, _st())
    assert rc == 0, lib().hnh_last_error_string()
    torch.cuda.synchronize()
    return _host_rows(ob, n, f, lddx, offset)


def finished(A, which, f):
    """The state after the finish: extremes of rows without entries set to 0."""
    A = A.copy()
    W = po.windows(A, which, f)
    for name in ("max", "min"):
        if name in which:
            W[name][W["c" + name] == 0] = 0.0
    return A


def close(got, want, tol):
    return np.abs(got - want).max() <= tol * max(np.abs(want).max(), 1.0)


def check_state(got, want, which, f, tol=1e-13):
    """Counts and extremes exactly, sums to rounding (the kernel fuses x * x + s)."""
    G, W = po.windows(got, which, f), po.windows(want, which, f)
    for k in W:
        if k in ("s1", "s2"):
            assert close(G[k], W[k], tol), k
        else:
            assert np.array_equal(G[k], W[k]), k


def grad_prep(A, dA, which, f):
    """D = [dS1 | dS2 | MAX | dMAX / CMAX | MIN | dMIN / CMIN] in numpy."""
    Dm = dA.copy()
    W, DW = po.windows(A, which, f), po.windows(Dm, which, f)
    for name in ("max", "min"):
        if name in which:
            c = W["c" + name]
            DW["c" + name][:] = np.divide(DW[name], c, out=np.zeros_like(c), where=c != 0)
            DW[name][:] = W[name]
    return Dm


def check_kernels(rowStart, col_idx, X, which, ld_step=(None, None), ld_grad=(None, None, None), offset=0):
    """The step from the initial state, the same over two blocks carrying the state, and the grad, against numpy."""
    n, f = len(rowStart) - 1, X.shape[1]
    rows = np.repeat(np.arange(n), np.diff(rowStart))
    want = po.multi_aggregate(rows, col_idx, n, X, which)
    A = run_step(rowStart, col_idx, X, initial_state(n, f, which), which, ld_step, offset)
    check_state(finished(A, which, f), want, which, f)
    # two blocks: the first half of every row's entries, then the rest, carrying the state (as ring steps do)
    k = np.arange(len(col_idx)) - rowStart[rows]
    first = k < np.diff(rowStart)[rows] // 2
    starts = [np.searchsorted(rows[m], np.arange(n + 1)).astype(np.int64) for m in (first, ~first)]
    A1 = run_step(starts[0], col_idx[first], X, initial_state(n, f, which), which, ld_step, offset)
    A2 = run_step(starts[1], col_idx[~first], X, A1, which, ld_step, offset)
    check_state(finished(A2, which, f), want, which, f)
    # grad on the transposed block (the rows of X are its stored rows)
    dA = np.random.default_rng(f + 2).standard_normal(want.shape)
    Dm = grad_prep(want, dA, which, f)
    order = np.lexsort((rows, col_idx))
    tr, tc = col_idx[order], rows[order]
    tStart = np.searchsorted(tr, np.arange(X.shape[0] + 1)).astype(np.int64)
    dX0 = np.random.default_rng(f + 3).standard_normal(X.shape)
    dX = run_grad(tStart, tc, X, Dm, dX0, which, ld_grad, offset)
    ref = dX0 + po.multi_aggregate_backward(rows, col_idx, X, want, dA, X.shape[0], which)
    assert close(dX, ref, 1e-12)
    assert np.array_equal(run_grad(tStart, tc, X, Dm, dX0, which, ld_grad, offset), dX)  # bit-identical repeats
    assert np.array_equal(run_step(rowStart, col_idx, X, initial_state(n, f, which), which, ld_step, offset), A)
    return want


def signed_zeros(X, rng):
    X = X.copy()
    X[(X == 0) & (rng.random(X.shape) < 0.5)] = -0.0
    return X


@pytest.mark.parametrize("which", SUBSETS)
@pytest.mark.parametrize("kind", ["normal", "relu", "int"])
@pytest.mark.parametrize("f", WIDTHS)
def test_kernels_match_numpy(world, f, kind, which):
    rng = np.random.default_rng(SEED + f)
    rowStart, col_idx = csr_block(rng, 300, 300)  # empty rows, duplicates, a hub row of 150 entries
    X = signed_zeros(inputs(rng, 300, f, kind), rng)
    A = check_kernels(rowStart, col_idx, X, which)
    if kind != "normal" and which != ("moments",):
        W = po.windows(A, which, f)
        assert max(W["c" + n].max() for n in ("max", "min") if n in which) > 1  # ties happened


@pytest.mark.parametrize("f", [4, 64, 256, 5, 602])
def test_kernels_odd_ld_and_misaligned_rows(world, f):
    rng = np.random.default_rng(SEED + 2 * f)
    rowStart, col_idx = csr_block(rng, 200, 200)
    X = inputs(rng, 200, f, "relu")
    w = 6 * f
    for lds, ldg, offset in (((f + 1, w), (f + 1, w, f), 0), ((f, w + 1), (f, w + 1, f), 0), ((f, w), (f, w, f + 1), 0),
                             ((f, w), (f, w, f), 1)):
        check_kernels(rowStart, col_idx, X, po.STATS, lds, ldg, offset)


@pytest.mark.parametrize("f,n", [(4, 200000), (64, 30000), (256, 12000), (5, 40000)])
def test_kernels_past_one_wave(world, f, n):
    rng = np.random.default_rng(SEED + n)
    rowStart, col_idx = csr_block(rng, n, n, per_row=3)
    check_kernels(rowStart, col_idx, inputs(rng, n, f, "int"), po.STATS)


@pytest.mark.parametrize("f", [64, 7])
def test_kernels_on_the_skewed_graph(world, f):
    rows, cols = skewed_tuples(4200, 4200, SEED)
    rows, cols = rows.astype(np.int64), cols.astype(np.int64)
    order = np.lexsort((cols, rows))
    rows, cols = rows[order], cols[order]
    rowStart = np.searchsorted(rows, np.arange(4201)).astype(np.int64)
    check_kernels(rowStart, cols, inputs(np.random.default_rng(SEED + f), 4200, f, "relu"), po.STATS)


def test_finish_and_grad_prep(world):
    f, which = 2, po.STATS
    A = np.array([[1.0, 2.0, 5.0, 9.0, -np.inf, 3.0, 0.0, 2.0, np.inf, 1.0, 0.0, 1.0]])
    Ad = torch.from_numpy(A.copy()).to(DEV)
    assert lib().hnh_multi_aggregate_finish_f64(Ad.data_ptr(), 12, 1, f, 7, _st()) == 0
    torch.cuda.synchronize()
    assert Ad.cpu().numpy().tolist() == [[1.0, 2.0, 5.0, 9.0, 0.0, 3.0, 0.0, 2.0, 0.0, 1.0, 0.0, 1.0]]
    dA = np.arange(12.0)[None, :] + 1
    dAd, Dd = torch.from_numpy(dA).to(DEV), torch.empty(1, 12, dtype=torch.float64, device=DEV)
    assert lib().hnh_multi_aggregate_grad_prep_f64(Ad.data_ptr(), 12, dAd.data_ptr(), 12, 1, f, 7, Dd.data_ptr(), 12, _st()) == 0
    torch.cuda.synchronize()
    want = grad_prep(finished(A, which, f), dA, which, f)
    assert np.array_equal(Dd.cpu().numpy(), want)


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


@pytest.mark.parametrize("which", [po.STATS, ("moments",), ("max", "min")])
@pytest.mark.parametrize("f", [8, 64, 13, 300])
@pytest.mark.parametrize("alg_name", ALGS)
def test_multi_aggregate_op(world, alg_name, f, which):
    N, rows, cols, alg, X = op_case(alg_name, f, "relu")
    nA, nB = alg.like_A_matrix().shape[0], alg.like_B_matrix().shape[0]
    w = D.Algorithm.multi_aggregate_width(which, f)
    Xd, A = D.Dense.create(nB, f), D.Dense.create(nA, w, 7.0)
    Xh = np.zeros((nB, f))
    Xh[:N] = X
    Xd.from_host(Xh)
    alg.multi_aggregate(Xd, A, which)
    want = po.multi_aggregate(rows, cols, N, X, which)
    got = A.to_host()
    check_state(got[:N], want, which, f)
    assert not got[9].any() and not got[N:].any()  # the empty row and the padding
    dAh = np.zeros((nA, w))
    dAh[:N] = np.random.default_rng(SEED + 6).standard_normal((N, w))
    dA, dX = D.Dense.create(nA, w), D.Dense.create(nB, f, 3.0)
    dA.from_host(dAh)
    ref = po.multi_aggregate_backward(rows, cols, X, want, dAh[:N], N, which)
    alg.multi_aggregate_backward(Xd, A, dA, dX, which)
    assert close(dX.to_host()[:N], ref, 1e-12)
    alg.multi_aggregate_backward(Xd, A, dA, dX, which, accumulate=True)
    assert close(dX.to_host()[:N], 2 * ref, 1e-12)
    A2 = D.Dense.create(nA, w)
    alg.multi_aggregate(Xd, A2, which)
    assert np.array_equal(A2.to_host(), got)


def test_multi_aggregate_refusals(world):
    N, rows, cols, alg, X = op_case("15d_fusion1", 8, "normal")
    nA, nB = alg.like_A_matrix().shape[0], alg.like_B_matrix().shape[0]
    Xd, A, dA, dX = D.Dense.create(nB, 8), D.Dense.create(nA, 48), D.Dense.create(nA, 48), D.Dense.create(nB, 8)
    for args, msg in (((Xd, Xd), "another operand|A-shaped"), ((D.Dense.create(nB, 0), A), "must be positive"),
                      ((Xd, D.Dense.create(nA, 47)), "A-shaped"), ((D.Dense.create(nB + 1, 8), A), "like_B_matrix")):
        with pytest.raises(RuntimeError, match=msg):
            alg.multi_aggregate(*args)
    assert lib().hnhd_alg_multi_aggregate(alg.h, Xd.h, A.h, 0) == -1 and b"selects no statistic" in lib().hnh_last_error_string()
    assert lib().hnhd_alg_multi_aggregate(alg.h, Xd.h, A.h, 8) == -1
    with pytest.raises(RuntimeError, match="another operand"):
        alg.multi_aggregate_backward(Xd, A, dA, Xd)
    with pytest.raises(RuntimeError, match="dX is"):
        alg.multi_aggregate_backward(Xd, A, dA, D.Dense.create(nB, 9))
    with pytest.raises(RuntimeError, match="A-shaped"):
        alg.multi_aggregate(Xd, A, ("moments",))


# ---- the model ----------------------------------------------------------------------------------------------------------
DEFAULT = (("mean", "min", "max", "std"), ("identity", "amplification", "attenuation"))
CONFIGS = {"default": DEFAULT, "all": (po.AGGREGATORS, po.SCALERS), "sum_var_lin": (("sum", "var"), ("linear", "inverse_linear")),
           "max_only": (("max",), ("identity",))}


def build(layers, cfg, logM=7, npr=5, alg_name="15d_fusion1", pattern=None, seed=SEED):
    aggs, scalers = cfg
    N = 1 << logM
    if pattern is None:
        rows, cols, _ = orc.er_tuples(logM, npr, seed)
    else:
        rows, cols = pattern
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    S = D.SpmatLocal.from_tuples(N, N, rows, cols, np.ones(len(rows)))
    alg = D.Algorithm(alg_name, S, layers[0][0], 1)
    hist = np.bincount(np.bincount(rows, minlength=N))
    net = D.PNA(alg, layers, aggregators=aggs, scalers=scalers, deg=hist)
    rng = np.random.default_rng(seed + 1)
    params = po.random_params(layers, len(aggs), len(scalers), rng)
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
    ocfg = (tuple(aggs), tuple(scalers)) + po.degree_averages(hist)
    return dict(N=N, rows=rows, cols=cols, alg=alg, net=net, params=params, X=X, G=G, layers=layers, cfg=ocfg)


def rel_err(got, ref):
    return np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-300)


def check_against_model(P, tol=1e-9):
    net, N, layers = P["net"], P["N"], P["layers"]
    net.forward()
    out, dX, dP = po.forward_backward(P["rows"], P["cols"], N, layers, P["params"], P["X"], P["G"][:N], *P["cfg"])
    assert np.abs(out).max() > 0
    assert rel_err(net.buffer(len(layers))[:N], out) < tol
    net.backward(P["G"])
    assert rel_err(net.input_grad()[:N], dX) < tol
    for l, grads in enumerate(dP):
        for name, g in grads.items():
            got = net.param_grad(l, name)
            assert got.shape == g.shape, (l, name)
            assert rel_err(got, g) < tol, (l, name, rel_err(got, g))


LAYER_SETS = {1: [(6, 4)], 2: [(6, 8), (8, 3)], 3: [(6, 8), (8, 5), (5, 4)]}


@pytest.mark.parametrize("cfg", list(CONFIGS))
@pytest.mark.parametrize("n_layers", [1, 2, 3])
def test_model_matches_oracle(world, n_layers, cfg):
    check_against_model(build(LAYER_SETS[n_layers], CONFIGS[cfg]))


@pytest.mark.parametrize("cfg", ["default", "all"])
@pytest.mark.parametrize("alg_name", ALGS)
def test_model_on_every_algorithm_with_duplicates_and_empty_rows(world, alg_name, cfg):
    rng = np.random.default_rng(SEED + 9)
    N = 128
    rows, cols = rng.integers(0, N, 500), rng.integers(0, N, 500)
    rows[rows % 7 == 0] = 1  # rows without entries and a hub row
    rows[:5], cols[:5] = 2, 11  # duplicates
    check_against_model(build([(6, 16), (16, 3)], CONFIGS[cfg], alg_name=alg_name, pattern=(rows, cols)))


def test_wide_input_layer(world):
    check_against_model(build([(300, 16), (16, 4)], DEFAULT, logM=8))


def test_backward_repeats_bit_identical_and_needs_a_forward(world):
    P = build(LAYER_SETS[2], CONFIGS["all"])
    net = P["net"]
    net.forward()
    net.backward(P["G"])
    first = [net.param_grad(l, n) for l in range(2) for n in net.param_names()] + [net.input_grad()]
    net.forward()
    net.backward(P["G"])
    again = [net.param_grad(l, n) for l in range(2) for n in net.param_names()] + [net.input_grad()]
    assert all(np.array_equal(a, b) for a, b in zip(first, again))
    net.set_param(0, "lin", P["params"][0]["lin"])
    with pytest.raises(RuntimeError, match="no forward pass"):
        net.backward(P["G"])


def flat_ok():
    return (C.c_int * 2)(6, 4)


def test_model_refusals(world):
    P = build(LAYER_SETS[1], DEFAULT)
    alg, net = P["alg"], P["net"]
    hist = [0, 3, 4]
    for aggs, msg in (((), "unknown name"), (("mean", "mean"), "appears twice"), (("lstm",), "unknown name")):
        with pytest.raises(RuntimeError, match=msg):
            D.PNA(alg, [(6, 4)], aggregators=aggs, deg=hist)
    for scalers, msg in ((("identity", "identity"), "appears twice"), (("log",), "unknown name")):
        with pytest.raises(RuntimeError, match=msg):
            D.PNA(alg, [(6, 4)], scalers=scalers, deg=hist)
    for bad in ([0, 0], [1, -2], np.ones((2, 2)), None):
        with pytest.raises(ValueError):
            D.PNA(alg, [(6, 4)], deg=bad)
    D.PNA(alg, [(6, 4)], scalers=("identity",))  # no scaler reads the histogram, so none is needed
    for bad in ([0, 0], [1, -2], np.ones((2, 2))):  # ... but one that is given is checked
        with pytest.raises(ValueError):
            D.PNA(alg, [(6, 4)], scalers=("identity",), deg=bad)
    assert lib().hnhd_pna_create(alg.h, 1, flat_ok(), b"mean", b"identity", float("nan"), 1.0, C.byref(C.c_void_p())) == -1
    assert b"NaN" in lib().hnh_last_error_string()
    out = C.c_void_p()
    flat = (C.c_int * 2)(6, 4)
    assert lib().hnhd_pna_create(alg.h, 1, flat, b"mean", b"linear", 0.0, 1.0, C.byref(out)) == -1
    assert b"delta_lin" in lib().hnh_last_error_string()
    assert lib().hnhd_pna_create(alg.h, 1, flat, b"mean", b"attenuation", 1.0, float("inf"), C.byref(out)) == -1
    assert b"delta_log" in lib().hnh_last_error_string()
    with pytest.raises(RuntimeError, match="does not take the width"):
        D.PNA(alg, [(6, 4), (5, 3)], deg=hist)
    with pytest.raises(RuntimeError, match="sizes must be positive"):
        D.PNA(alg, [(6, 0)], deg=hist)
    with pytest.raises(RuntimeError, match="no parameter"):
        net.param_shape(0, "root")
    with pytest.raises(RuntimeError, match="no such layer"):
        net.param(1, "lin")
    with pytest.raises(RuntimeError, match="no dropout"):
        net._forward(0.1, 0)
    assert net.param_shape(0, "pre") == (12, 6) and net.param_shape(0, "post") == (78, 4) and net.param_shape(0, "lin_bias") == (4,)


# ---- training -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cfg", ["default", "all"])
def test_train_step_matches_torch_adamw(world, cfg):
    P = build([(6, 8), (8, 3)], CONFIGS[cfg])
    N = P["N"]
    rng = np.random.default_rng(SEED + 11)
    labels = rng.integers(0, 3, N)
    labels[rng.random(N) < 0.3] = -1
    lab = np.full(P["net"].buffer_shape(2)[0], -1)
    lab[:N] = labels
    L = D.NodeLabels(P["net"], lab, 3)
    opt = D.AdamW(lr=1e-2, max_grad_norm=0.5)
    got = [P["net"].train_step(L, opt) for _ in range(4)]
    res, trained = po.train(P["rows"], P["cols"], N, P["layers"], P["params"], P["X"], P["cfg"], labels, 4, lr=1e-2, max_grad_norm=0.5)
    for g, w in zip(got, res):
        assert abs(g.loss - w[0]) <= 1e-9 * abs(w[0]) and abs(g.grad_norm - w[3]) <= 1e-9 * abs(w[3])
        assert (g.correct, g.labelled) == (w[1], w[2])
    for l, Pt in enumerate(trained):
        for k, v in Pt.items():
            assert close(P["net"].param(l, k), v, 1e-9), (l, k)


def test_link_train_step_matches_torch_adamw(world):
    P = build([(6, 8), (8, 4)], DEFAULT)
    N = P["N"]
    rng = np.random.default_rng(SEED + 12)
    tr, tc = rng.integers(0, N, 4 * N), rng.integers(0, N, 4 * N)
    y = rng.choice([0.0, 1.0], 4 * N)
    algT = D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, tr, tc, y), 6, 1)
    t = D.LinkTargets(P["net"], algT)
    opt = D.AdamW(lr=1e-2)
    got = [P["net"].link_train_step(t, opt) for _ in range(3)]
    res, trained = po.train_link(P["rows"], P["cols"], N, P["layers"], P["params"], P["X"], P["cfg"], (tr, tc, y), 3, lr=1e-2)
    for g, w in zip(got, res):
        assert abs(g.loss - w[0]) <= 1e-9 * abs(w[0]) and abs(g.grad_norm - w[3]) <= 1e-9 * abs(w[3])
        assert g.labelled == w[2] and abs(g.correct - w[1]) <= 1
    for l, Pt in enumerate(trained):
        for k, v in Pt.items():
            assert close(P["net"].param(l, k), v, 1e-9), (l, k)


@pytest.mark.parametrize("pool", gro.POOLS)
def test_graph_train_step_matches_torch_adamw(world, pool):
    P = build([(6, 8), (8, 4)], DEFAULT)
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
    tp = [{k: po._t(v).clone().requires_grad_() for k, v in Pd.items()} for Pd in P["params"]]
    x = po._t(P["X"])
    want, head = gro.train(lambda t: po.model_torch(P["rows"], P["cols"], N, P["layers"], tp, x, *P["cfg"]),
                           [v for Pd in tp for v in Pd.values()], batch[:N], G, pool, (W, b), labels, 3, lr=1e-2, max_grad_norm=0.5)
    for g, w in zip(got, want):
        assert abs(g.loss - w[0]) <= 1e-9 * abs(w[0]) and abs(g.grad_norm - w[3]) <= 1e-9 * abs(w[3]), (g, w)
        assert (g.correct, g.labelled) == (w[1], w[2])
    for l, Pd in enumerate(tp):
        for k, v in Pd.items():
            assert close(net.param(l, k), v.detach().numpy(), 1e-9), (l, k)
    assert close(ro.param("weight"), head[0], 1e-9) and close(ro.param("bias"), head[1], 1e-9)


def _spread_batch(G, seed):
    """Graphs of 6 centre nodes and 12 leaves.  Centre j aggregates leaves 2j and 2j + 1 (the leaves aggregate nothing);
    a graph of label 1 gives each leaf pair the features (+1, -1), one of label 0 gives them (0, 0).  Every node's first
    feature is 1 and the readout pools the centre nodes only, so the centres' own features and the mean of their
    neighbours are the same for both labels: only the spread of the neighbours (var, std, min, max) tells them apart."""
    rng = np.random.default_rng(seed)
    n = 18
    N = G * n
    labels = np.repeat([0, 1], G // 2)
    rng.shuffle(labels)
    rows, cols, feats = [], [], np.zeros((N, 2))
    feats[:, 0] = 1.0
    for g in range(G):
        base = g * n
        for j in range(6):
            rows += [base + j, base + j]
            cols += [base + 6 + 2 * j, base + 7 + 2 * j]
            if labels[g]:
                feats[base + 6 + 2 * j, 1], feats[base + 7 + 2 * j, 1] = 1.0, -1.0
    batch = np.full(N, -1, np.int64)
    for g in range(G):
        batch[g * n:g * n + 6] = g
    return N, np.array(rows), np.array(cols), feats, batch, labels


@pytest.mark.parametrize("aggs,learns", [(("mean", "std"), True), (("mean",), False)])
def test_learning_neighbourhood_spread(world, aggs, learns):
    """A graph train step learns a label that only the neighbourhood spread carries with std, and cannot without it."""
    G = 64
    N, rows, cols, feats, batch, labels = _spread_batch(G, SEED + 14)
    S = D.SpmatLocal.from_tuples(N, N, rows, cols, np.ones(len(rows)))
    alg = D.Algorithm("15d_fusion1", S, 2, 1)
    layers = [(2, 16)]
    net = D.PNA(alg, layers, aggregators=aggs, scalers=("identity",))
    for l, Pd in enumerate(po.random_params(layers, len(aggs), 1, np.random.default_rng(SEED + 15))):
        for k, v in Pd.items():
            net.set_param(l, k, v)
    Xl = np.zeros(net.buffer_shape(0))
    Xl[:N] = feats
    net.set_input(Xl)
    b = np.full(net.buffer_shape(1)[0], -1, np.int64)
    b[:N] = batch
    ro = D.GraphReadout(net, b, G, pool="mean", num_classes=2)
    gl = D.GraphLabels(ro, labels, 2)
    opt = D.AdamW(lr=1e-2)
    steps = [net.graph_train_step(ro, gl, opt) for _ in range(150)]
    if learns:
        assert steps[-1].loss < 0.5 * steps[0].loss and steps[-1].correct >= 0.9 * G, (steps[0], steps[-1])
    else:  # every centre row is the same in both labels: no better than the balanced prior
        _, _, _, logits = net.graph_evaluate(ro, gl)
        assert np.abs(logits - logits[0]).max() <= 1e-12 * max(np.abs(logits).max(), 1.0)
        assert steps[-1].correct <= G // 2
