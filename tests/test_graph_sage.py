"""GraphSAGE, CPU side: the fp64 oracle (tests/graph_sage_oracle.py) against finite differences for every aggregator,
against PyG's SAGEConv formula written out by hand, the max backward on hand-built ties, duplicates and empty rows, and
the new C and Python entry points refuse bad arguments without a GPU."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import graph_sage_oracle as gso
from tests.test_sparse_attention_bias import _pattern

LAYERS = [(3, 4), (4, 2)]


@pytest.mark.parametrize("aggr", gso.AGGREGATIONS)
def test_oracle_gradcheck(aggr):
    rng = np.random.default_rng(7)
    N = 9
    rows, cols = _pattern(rng, N, N, per_row=3)
    rows, cols = np.append(rows, [2, 2]), np.append(cols, [5, 5])  # a duplicate
    params = gso.random_params(LAYERS, rng)
    tp = [{k: gso._t(v).clone().requires_grad_() for k, v in P.items()} for P in params]
    # continuous inputs: no ties and no ReLU kinks at the evaluation point, so the model is smooth there
    x = gso._t(rng.standard_normal((N, 3))).requires_grad_()
    leaves = [x] + [v for P in tp for v in P.values()]

    def f(*args):
        xx, flat = args[0], list(args[1:])
        P = [{k: flat.pop(0) for k in ("neigh", "neigh_bias", "root")} for _ in LAYERS]
        return gso.model_torch(rows, cols, N, LAYERS, P, xx, aggr)

    assert torch.autograd.gradcheck(f, tuple(leaves), eps=1e-6, atol=1e-7)


def test_oracle_is_sageconv():
    """Y = lin_l(aggr(x)) + lin_r(x) with the aggregations written out row by row."""
    rng = np.random.default_rng(3)
    N, f, r = 7, 3, 2
    rows, cols = np.array([0, 0, 0, 1, 3, 3, 6]), np.array([1, 2, 2, 0, 4, 5, 6])  # row 0 holds a duplicate
    X = rng.standard_normal((N, f))
    P = gso.random_params([(f, r)], rng)[0]
    for aggr in gso.AGGREGATIONS:
        A = np.zeros((N, f))
        for u in range(N):
            vs = cols[rows == u]
            if len(vs):
                A[u] = {"sum": X[vs].sum(0), "mean": X[vs].mean(0), "max": X[vs].max(0)}[aggr]
        want = A @ P["neigh"] + P["neigh_bias"] + X @ P["root"]
        got = gso.model_torch(rows, cols, N, [(f, r)], [{k: gso._t(v) for k, v in P.items()}], gso._t(X), aggr).numpy()
        assert np.allclose(got, want, rtol=1e-14, atol=1e-14), aggr
        if aggr == "max":
            Z, Cn = gso.max_aggregate(rows, cols, N, X)
            assert np.array_equal(Z, A) and Cn[2].sum() == 0 and Cn[0].min() >= 1


def test_max_backward_splits_ties_and_counts_duplicates():
    # row 0: entries 1, 2, 2 (a duplicate); row 1: entry 3; row 2: no entries; row 3: entries 0, 4
    rows, cols = np.array([0, 0, 0, 1, 3, 3]), np.array([1, 2, 2, 3, 0, 4])
    X = np.array([[0.0, 1.0],
                  [5.0, 2.0],
                  [5.0, 7.0],
                  [-1.0, -0.0],
                  [0.0, 3.0]])
    Z, Cn = gso.max_aggregate(rows, cols, 4, X)
    assert np.array_equal(Z, [[5.0, 7.0], [-1.0, 0.0], [0.0, 0.0], [0.0, 3.0]])
    # column 0 of row 0: X[1] and both copies of X[2] tie at 5; column 0 of row 3: X[0] and X[4] tie at 0
    assert np.array_equal(Cn, [[3.0, 2.0], [1.0, 1.0], [0.0, 0.0], [2.0, 1.0]])
    dZ = np.array([[6.0, 10.0], [1.0, 2.0], [100.0, 100.0], [4.0, 8.0]])
    dX = gso.max_aggregate_backward(rows, cols, Z, Cn, dZ, 5, X)
    want = np.array([[2.0, 0.0],      # row 3's tie at 0: 4 / 2
                     [2.0, 0.0],      # one of row 0's three: 6 / 3
                     [4.0, 10.0],     # twice (the duplicate): 2 x 6 / 3, and 2 x 10 / 2 in column 1
                     [1.0, 2.0],
                     [2.0, 8.0]])
    assert np.array_equal(dX, want)
    # the torch model gives the same
    x = torch.from_numpy(X).requires_grad_()
    A = gso.aggregate_torch(rows, cols, 4, x, "max")
    assert np.array_equal(A.detach().numpy(), Z)
    (A * torch.from_numpy(dZ)).sum().backward()
    assert np.array_equal(x.grad.numpy(), want)
    # torch's autograd of scatter_reduce(include_self=False) agrees wherever the maximum is not 0; at a maximum of exactly
    # 0 it counts the untouched zero of `self` as one more tie (row 3, column 0; row 1, column 1)
    x = torch.from_numpy(X).requires_grad_()
    index = torch.from_numpy(rows)[:, None].expand(len(rows), 2)
    A = torch.zeros(4, 2, dtype=torch.float64).scatter_reduce(0, index, x[torch.from_numpy(cols)], "amax", include_self=False)
    (A * torch.from_numpy(dZ)).sum().backward()
    at_zero = np.zeros_like(want, bool)
    at_zero[[0, 4], 0] = at_zero[3, 1] = True
    assert np.array_equal(x.grad.numpy()[~at_zero], want[~at_zero])
    assert np.allclose(x.grad.numpy()[at_zero], [4 / 3, 2 / 2, 4 / 3])


def test_max_ties_of_signed_zeros():
    rows, cols = np.array([0, 0]), np.array([0, 1])
    X = np.array([[-0.0], [0.0]])
    Z, Cn = gso.max_aggregate(rows, cols, 1, X)
    assert Z[0, 0] == 0.0 and Cn[0, 0] == 2.0
    dX = gso.max_aggregate_backward(rows, cols, Z, Cn, np.array([[1.0]]), 2, X)
    assert np.array_equal(dX, [[0.5], [0.5]])


def test_max_kernels_validate_without_a_gpu(hnh):
    bufs = [(C.c_double * 64)() for _ in range(8)]
    rs, ci, x, z, c, g, dx, dz = (C.addressof(b) for b in bufs)

    def step(rs=rs, ci=ci, rows=4, nnz=4, x=x, ldx=4, f=4, z=z, ldz=4, c=c, ldc=4):
        return hnh.hnh_max_aggregate_step_f64(rs, ci, rows, nnz, x, ldx, f, z, ldz, c, ldc, None)

    def grad(rs=rs, ci=ci, rows=4, nnz=4, x=x, ldx=4, z=z, ldz=4, g=g, ldg=4, f=4, dx=dx, lddx=4):
        return hnh.hnh_max_aggregate_grad_f64(rs, ci, rows, nnz, x, ldx, z, ldz, g, ldg, f, dx, lddx, None)

    assert step(rows=-1) == -1 and b"negative" in hnh.hnh_last_error_string()
    assert step(f=0) == -1 and b"f must be positive" in hnh.hnh_last_error_string()
    for kw in (dict(ldx=3), dict(ldz=3), dict(ldc=3)):
        assert step(**kw) == -1 and b"leading dimension" in hnh.hnh_last_error_string(), kw
    for k in ("rs", "ci", "x", "z", "c"):
        assert step(**{k: None}) == -1 and b"null" in hnh.hnh_last_error_string(), k
    assert step(z=x) == -1 and b"may not be the input" in hnh.hnh_last_error_string()
    assert step(c=z) == -1 and b"distinct" in hnh.hnh_last_error_string()
    assert step(rows=0) == 0 and step(nnz=0, rs=None) == 0  # empty blocks are a no-op
    assert grad(nnz=-1) == -1 and grad(f=-3) == -1
    for kw in (dict(ldx=3), dict(ldz=3), dict(ldg=3), dict(lddx=3)):
        assert grad(**kw) == -1 and b"leading dimension" in hnh.hnh_last_error_string(), kw
    for k in ("rs", "ci", "x", "z", "g", "dx"):
        assert grad(**{k: None}) == -1 and b"null" in hnh.hnh_last_error_string(), k
    for k in ("x", "z", "g"):
        assert grad(dx={"x": x, "z": z, "g": g}[k]) == -1 and b"may not be an input" in hnh.hnh_last_error_string()
    assert grad(rows=0) == 0 and grad(nnz=0, dx=None) == 0
    assert hnh.hnh_max_aggregate_finish_f64(z, c, -1, None) == -1 and hnh.hnh_max_aggregate_finish_f64(None, c, 4, None) == -1
    assert hnh.hnh_max_aggregate_finish_f64(z, z, 4, None) == -1 and hnh.hnh_max_aggregate_finish_f64(None, None, 0, None) == 0
    assert hnh.hnh_max_aggregate_grad_scale_f64(g, dz, c, -1, None) == -1
    assert hnh.hnh_max_aggregate_grad_scale_f64(g, None, c, 4, None) == -1
    assert hnh.hnh_max_aggregate_grad_scale_f64(c, dz, c, 4, None) == -1 and b"may not be C" in hnh.hnh_last_error_string()
    if not torch.cuda.is_available():  # no CPU fallback: compute fails with HNH_E_CUDA
        assert step() == -2 and grad() == -2
        assert hnh.hnh_max_aggregate_finish_f64(z, c, 4, None) == -2
        assert hnh.hnh_max_aggregate_grad_scale_f64(g, dz, c, 4, None) == -2


def test_sage_driver_entry_points_validate_without_a_gpu(hnh):
    out = C.c_void_p()
    res = (C.c_double * 4)()
    p = C.addressof(res)
    layers = (C.c_int * 4)(3, 4, 4, 2)
    assert hnh.hnhd_sage_create(None, 2, layers, b"mean", C.byref(out)) == -1 and b"bad argument" in hnh.hnh_last_error_string()
    assert hnh.hnhd_sage_create(p, 0, layers, b"mean", C.byref(out)) == -1
    assert hnh.hnhd_sage_create(p, 2, None, b"mean", C.byref(out)) == -1
    assert hnh.hnhd_sage_create(p, 2, layers, None, C.byref(out)) == -1
    assert hnh.hnhd_sage_create(p, 2, layers, b"mean", None) == -1
    r, c = C.c_int64(), C.c_int64()
    assert hnh.hnhd_sage_param_shape(None, 0, b"neigh", C.byref(r), C.byref(c)) == -1
    assert hnh.hnhd_sage_set_param(None, 0, b"root", p) == -1 and hnh.hnhd_sage_get_param(None, 0, b"root", p) == -1
    assert hnh.hnhd_sage_get_param_grad(None, 0, b"root", p) == -1
    assert hnh.hnhd_sage_buffer_shape(None, 0, C.byref(r), C.byref(c)) == -1
    assert hnh.hnhd_sage_set_input(None, p) == -1 and hnh.hnhd_sage_get_buffer(None, 0, p) == -1
    assert hnh.hnhd_sage_forward(None) == -1 and hnh.hnhd_sage_backward(None, p) == -1
    assert hnh.hnhd_sage_get_input_grad(None, p) == -1
    for args in ((None, p, p), (p, None, p), (p, p, None)):
        assert hnh.hnhd_sage_train_step(*args, res) == -1 and b"null" in hnh.hnh_last_error_string()
        assert hnh.hnhd_sage_link_train_step(*args, res) == -1 and b"null" in hnh.hnh_last_error_string()
    assert hnh.hnhd_sage_train_step(p, p, p, None) == -1
    assert hnh.hnhd_sage_link_evaluate(None, p, None, res) == -1 and hnh.hnhd_sage_link_evaluate(p, None, None, res) == -1
    assert hnh.hnhd_sage_link_evaluate(p, p, None, None) == -1
    hnh.hnhd_sage_destroy(None)
    for args in ((None, p, p, p), (p, None, p, p), (p, p, None, p), (p, p, p, None)):
        assert hnh.hnhd_alg_max_aggregate(*args) == -1 and b"null" in hnh.hnh_last_error_string()
    for i in range(6):
        args = [p] * 6
        args[i] = None
        assert hnh.hnhd_alg_max_aggregate_backward(*args, 0) == -1 and b"null" in hnh.hnh_last_error_string()


def test_python_front_end_validates_sage_arguments():
    from distributed_sddmm_b200 import driver as D
    alg = D.Algorithm.__new__(D.Algorithm)
    alg.h = None
    with pytest.raises(ValueError, match="aggr"):
        D.GraphSAGE(alg, [(3, 4)], aggr="lstm")
    with pytest.raises(ValueError, match="pairs"):
        D.GraphSAGE(alg, [(3, 4, 2)])
    with pytest.raises(ValueError, match="pairs"):
        D.GraphSAGE(alg, [])
    with pytest.raises(RuntimeError, match="sage_create failed"):
        D.GraphSAGE(alg, [(3, 4)], aggr="max")  # null algorithm handle
    with pytest.raises(TypeError, match="X must be a Dense"):
        alg.max_aggregate(np.zeros((2, 2)), None, None)
    dense = D.Dense.__new__(D.Dense)
    dense.h = None
    with pytest.raises(TypeError, match="dX must be a Dense"):
        alg.max_aggregate_backward(dense, dense, dense, dense, np.zeros(2))
    with pytest.raises(RuntimeError, match="max_aggregate failed"):
        alg.max_aggregate(dense, dense, dense)
    net = D.GraphSAGE.__new__(D.GraphSAGE)
    net.h = None
    opt = D.AdamW()
    with pytest.raises(TypeError, match="NodeLabels"):
        net.train_step(None, opt)
    with pytest.raises(TypeError, match="LinkTargets"):
        net.link_train_step(None, opt)
    with pytest.raises(TypeError, match="LinkTargets"):
        net.link_evaluate(object())
    targets = D.LinkTargets.__new__(D.LinkTargets)
    targets.h = None
    with pytest.raises(TypeError, match="AdamW"):
        net.link_train_step(targets, None)
    with pytest.raises(RuntimeError, match="sage_param_shape failed"):
        net.param_shape(0, "neigh")
