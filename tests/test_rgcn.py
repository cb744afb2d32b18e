"""R-GCN, CPU side: the fp64 oracle (tests/rgcn_oracle.py) against finite differences for both aggregators, against the
GraphSAGE mean oracle at one relation, on duplicate pairs of different relations written out by hand, the numpy kernels
against the torch model, and the new C and Python entry points refuse bad arguments without a GPU."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import graph_sage_oracle as gso
from tests import rgcn_oracle as ro
from tests.test_sparse_attention_bias import _pattern

LAYERS = [(3, 4), (4, 2)]


@pytest.mark.parametrize("aggr", ro.AGGREGATIONS)
def test_oracle_gradcheck(aggr):
    rng = np.random.default_rng(7)
    N, R = 9, 3
    rows, cols = _pattern(rng, N, N, per_row=3)
    rows, cols = np.append(rows, [2, 2]), np.append(cols, [5, 5])  # a duplicate pair
    rels = rng.integers(0, R, len(rows)).astype(np.float64)
    rels[-2:] = [0, 2]  # ... under two relations
    params = ro.random_params(LAYERS, R, rng)
    tp = [{k: ro._t(v).clone().requires_grad_() for k, v in P.items()} for P in params]
    x = ro._t(rng.standard_normal((N, 3))).requires_grad_()
    leaves = [x] + [v for P in tp for v in P.values()]

    def f(*args):
        xx, flat = args[0], list(args[1:])
        P = [{k: flat.pop(0) for k in ro.PARAMS} for _ in LAYERS]
        return ro.model_torch(rows, cols, rels, N, LAYERS, P, xx, R, aggr)

    assert torch.autograd.gradcheck(f, tuple(leaves), eps=1e-6, atol=1e-7)


def test_one_relation_mean_is_sage_mean():
    rng = np.random.default_rng(3)
    N = 11
    rows, cols = _pattern(rng, N, N, per_row=4)
    rows, cols = np.append(rows, [1, 1]), np.append(cols, [4, 4])
    params = ro.random_params(LAYERS, 1, rng)
    X = rng.standard_normal((N, 3))
    got = ro.model_torch(rows, cols, np.zeros(len(rows)), N, LAYERS, [{k: ro._t(v) for k, v in P.items()} for P in params],
                         ro._t(X), 1, "mean")
    sage = [{"neigh": ro._t(P["weight"]), "neigh_bias": ro._t(P["bias"]), "root": ro._t(P["root"])} for P in params]
    want = gso.model_torch(rows, cols, N, LAYERS, sage, ro._t(X), "mean")
    assert np.allclose(got.numpy(), want.numpy(), rtol=1e-13, atol=1e-13)


def test_duplicate_pairs_under_different_relations():
    # row 0: (0, 1) under relations 0 and 1, (0, 2) under relation 1; row 1: (1, 2) under relation 0 and an entry whose
    # value is no relation; row 2: nothing
    rows, cols = np.array([0, 0, 0, 1, 1]), np.array([1, 1, 2, 2, 0])
    rels = np.array([0.0, 1.0, 1.0, 0.0, 0.5])
    X = np.array([[1.0, -2.0], [3.0, 5.0], [7.0, 11.0]])
    R, f, r = 2, 2, 3
    A = ro.relational_aggregate(rows, cols, rels, 3, X, R)
    assert np.array_equal(A, [[3.0, 5.0, 10.0, 16.0], [7.0, 11.0, 0.0, 0.0], [0.0, 0.0, 0.0, 0.0]])
    assert np.array_equal(ro.relation_counts(rows, rels, 3, R), [[1, 2], [1, 0], [0, 0]])
    P = ro.random_params([(f, r)], R, np.random.default_rng(1))[0]
    W = P["weight"].reshape(R, f, r)
    for aggr, Ab in (("sum", A), ("mean", A / np.maximum(ro.relation_counts(rows, rels, 3, R), 1).repeat(f, 1))):
        want = Ab[:, :f] @ W[0] + Ab[:, f:] @ W[1] + X @ P["root"] + P["bias"]
        got = ro.model_torch(rows, cols, rels, 3, [(f, r)], [{k: ro._t(v) for k, v in P.items()}], ro._t(X), R, aggr)
        assert np.allclose(got.numpy(), want, rtol=1e-14, atol=1e-14), aggr
    dA = np.arange(12.0).reshape(3, 4)
    # dX[1] takes row 0's windows of relations 0 and 1, dX[2] row 0's relation 1 and row 1's relation 0
    assert np.array_equal(ro.relational_aggregate_backward(rows, cols, rels, dA, 3, R), [[0, 0], [2, 4], [6, 8]])


def test_numpy_kernels_match_the_torch_model():
    """The numpy kernels against the torch model read through a weight that selects one relation's window; values that
    are no relation (-1, R, 0.5, NaN, +-inf) count nowhere in either."""
    rng = np.random.default_rng(5)
    N, R, f = 13, 4, 3
    rows, cols = _pattern(rng, N, N, per_row=5)
    rels = rng.integers(0, R, len(rows)).astype(np.float64)
    rels[::7] = np.resize([-1.0, R, 0.5, np.nan, np.inf, -np.inf], len(rels[::7]))
    X = ro._t(rng.standard_normal((N, f))).requires_grad_()
    dA = rng.standard_normal((N, R * f))
    A = ro.relational_aggregate(rows, cols, rels, N, X.detach().numpy(), R)
    loss = 0
    for rho in range(R):
        W = torch.zeros(R * f, f, dtype=torch.float64)
        W[rho * f:(rho + 1) * f] = torch.eye(f, dtype=torch.float64)
        P = [{"weight": W, "bias": torch.zeros(f, dtype=torch.float64), "root": torch.zeros(f, f, dtype=torch.float64)}]
        got = ro.model_torch(rows, cols, rels, N, [(f, f)], P, X, R, "sum")
        assert np.allclose(got.detach().numpy(), A[:, rho * f:(rho + 1) * f], rtol=1e-14, atol=1e-14)
        loss = loss + (got * ro._t(dA[:, rho * f:(rho + 1) * f])).sum()
    loss.backward()
    assert np.allclose(ro.relational_aggregate_backward(rows, cols, rels, dA, N, R), X.grad.numpy(), rtol=1e-13, atol=1e-13)


def test_relational_kernels_validate_without_a_gpu(hnh):
    bufs = [(C.c_double * 64)() for _ in range(6)]
    rs, ci, v, x, a, cn = (C.addressof(b) for b in bufs)

    def agg(rs=rs, ci=ci, v=v, rows=4, nnz=4, x=x, ldx=4, f=4, R=2, a=a, lda=8):
        return hnh.hnh_relational_aggregate_f64(rs, ci, v, rows, nnz, x, ldx, f, R, a, lda, None)

    def grad(rs=rs, ci=ci, v=v, rows=4, nnz=4, da=a, ldda=8, f=4, R=2, dx=x, lddx=4):
        return hnh.hnh_relational_aggregate_grad_f64(rs, ci, v, rows, nnz, da, ldda, f, R, dx, lddx, None)

    for fn in (agg, grad):
        assert fn(rows=-1) == -1 and b"negative" in hnh.hnh_last_error_string()
        assert fn(f=0) == -1 and b"f must be positive" in hnh.hnh_last_error_string()
        assert fn(R=0) == -1 and b"relation count" in hnh.hnh_last_error_string()
        assert fn(R=1 << 20, f=1 << 12) == -1 and b"below 2^31" in hnh.hnh_last_error_string()
        assert fn(rows=0) == 0 and fn(nnz=0, rs=None) == 0  # empty blocks are a no-op
        for k in ("rs", "ci", "v"):
            assert fn(**{k: None}) == -1 and b"null" in hnh.hnh_last_error_string(), k
    for kw in (dict(ldx=3), dict(lda=7)):
        assert agg(**kw) == -1 and b"leading dimension" in hnh.hnh_last_error_string(), kw
    for kw in (dict(ldda=7), dict(lddx=3)):
        assert grad(**kw) == -1 and b"leading dimension" in hnh.hnh_last_error_string(), kw
    assert agg(x=None) == -1 and agg(a=None) == -1 and grad(da=None) == -1 and grad(dx=None) == -1
    assert agg(a=x, lda=8, ldx=8) == -1 and b"may not be an input" in hnh.hnh_last_error_string()
    assert agg(a=v) == -1 and grad(dx=v) == -1 and grad(dx=a, lddx=8) == -1
    ws = hnh.hnh_window_scale_f64
    assert ws(a, 8, cn, 2, -1, 4, 2, None) == -1 and ws(a, 8, cn, 2, 4, 0, 2, None) == -1 and ws(a, 8, cn, 2, 4, 4, 0, None) == -1
    assert ws(a, 7, cn, 2, 4, 4, 2, None) == -1 and ws(a, 8, cn, 1, 4, 4, 2, None) == -1
    assert ws(None, 8, cn, 2, 4, 4, 2, None) == -1 and ws(a, 8, None, 2, 4, 4, 2, None) == -1
    assert ws(a, 8, a, 8, 4, 4, 2, None) == -1 and b"may not be C" in hnh.hnh_last_error_string()
    assert ws(None, 8, None, 2, 0, 4, 2, None) == 0
    rc = hnh.hnh_relation_check_f64
    assert rc(cn, v, -1, 2, None) == -1 and rc(cn, v, 4, 0, None) == -1
    assert rc(None, v, 4, 2, None) == -1 and rc(cn, None, 4, 2, None) == -1 and rc(cn, None, 0, 2, None) == 0
    if not torch.cuda.is_available():  # no CPU fallback: compute fails with HNH_E_CUDA
        assert agg() == -2 and grad() == -2
        assert ws(a, 8, cn, 2, 4, 4, 2, None) == -2 and rc(cn, v, 4, 2, None) == -2


def test_rgcn_driver_entry_points_validate_without_a_gpu(hnh):
    out = C.c_void_p()
    res = (C.c_double * 4)()
    p = C.addressof(res)
    layers = (C.c_int * 4)(3, 4, 4, 2)
    assert hnh.hnhd_rgcn_create(None, 2, layers, 3, b"mean", C.byref(out)) == -1 and b"bad argument" in hnh.hnh_last_error_string()
    assert hnh.hnhd_rgcn_create(p, 0, layers, 3, b"mean", C.byref(out)) == -1
    assert hnh.hnhd_rgcn_create(p, 2, None, 3, b"mean", C.byref(out)) == -1
    assert hnh.hnhd_rgcn_create(p, 2, layers, 3, None, C.byref(out)) == -1
    assert hnh.hnhd_rgcn_create(p, 2, layers, 3, b"mean", None) == -1
    # refused before the algorithm is touched
    assert hnh.hnhd_rgcn_create(p, 2, layers, 0, b"mean", C.byref(out)) == -1 and b"relation count" in hnh.hnh_last_error_string()
    assert hnh.hnhd_rgcn_create(p, 2, layers, 3, b"max", C.byref(out)) == -1
    assert b"unknown aggregation" in hnh.hnh_last_error_string()
    bad = (C.c_int * 4)(3, 4, 5, 2)
    assert hnh.hnhd_rgcn_create(p, 2, bad, 3, b"sum", C.byref(out)) == -1 and b"does not take the width" in hnh.hnh_last_error_string()
    zero = (C.c_int * 2)(3, 0)
    assert hnh.hnhd_rgcn_create(p, 1, zero, 3, b"sum", C.byref(out)) == -1 and b"sizes must be positive" in hnh.hnh_last_error_string()
    wide = (C.c_int * 2)(1 << 20, 4)
    assert hnh.hnhd_rgcn_create(p, 1, wide, 1 << 12, b"sum", C.byref(out)) == -1 and b"below 2^31" in hnh.hnh_last_error_string()
    r, c = C.c_int64(), C.c_int64()
    assert hnh.hnhd_rgcn_param_shape(None, 0, b"weight", C.byref(r), C.byref(c)) == -1
    assert hnh.hnhd_rgcn_set_param(None, 0, b"root", p) == -1 and hnh.hnhd_rgcn_get_param(None, 0, b"root", p) == -1
    assert hnh.hnhd_rgcn_get_param_grad(None, 0, b"root", p) == -1
    assert hnh.hnhd_rgcn_buffer_shape(None, 0, C.byref(r), C.byref(c)) == -1
    assert hnh.hnhd_rgcn_set_input(None, p) == -1 and hnh.hnhd_rgcn_get_buffer(None, 0, p) == -1
    assert hnh.hnhd_rgcn_forward(None) == -1 and hnh.hnhd_rgcn_backward(None, p) == -1
    assert hnh.hnhd_rgcn_get_input_grad(None, p) == -1
    for args in ((None, p, p), (p, None, p), (p, p, None)):
        assert hnh.hnhd_rgcn_train_step(*args, res) == -1 and b"null" in hnh.hnh_last_error_string()
        assert hnh.hnhd_rgcn_link_train_step(*args, res) == -1 and b"null" in hnh.hnh_last_error_string()
    assert hnh.hnhd_rgcn_train_step(p, p, p, None) == -1
    assert hnh.hnhd_rgcn_link_evaluate(None, p, None, res) == -1 and hnh.hnhd_rgcn_link_evaluate(p, None, None, res) == -1
    assert hnh.hnhd_rgcn_link_evaluate(p, p, None, None) == -1
    hnh.hnhd_rgcn_destroy(None)
    for args in ((None, p, p), (p, None, p), (p, p, None)):
        assert hnh.hnhd_alg_relational_aggregate(*args, 2) == -1 and b"null" in hnh.hnh_last_error_string()
        assert hnh.hnhd_alg_relational_aggregate_backward(*args, 2, 0) == -1 and b"null" in hnh.hnh_last_error_string()


def test_python_front_end_validates_rgcn_arguments():
    from distributed_sddmm_b200 import driver as D
    alg = D.Algorithm.__new__(D.Algorithm)
    alg.h = None
    with pytest.raises(ValueError, match="aggr"):
        D.RGCN(alg, [(3, 4)], num_relations=2, aggr="max")
    with pytest.raises(ValueError, match="num_relations"):
        D.RGCN(alg, [(3, 4)], num_relations=0)
    with pytest.raises(ValueError, match="pairs"):
        D.RGCN(alg, [(3, 4, 2)], num_relations=2)
    with pytest.raises(ValueError, match="pairs"):
        D.RGCN(alg, [], num_relations=2)
    with pytest.raises(ValueError, match="do not chain"):
        D.RGCN(alg, [(3, 4), (5, 2)], num_relations=2)
    with pytest.raises(RuntimeError, match="rgcn_create failed"):
        D.RGCN(alg, [(3, 4)], num_relations=2)  # null algorithm handle
    with pytest.raises(TypeError, match="X must be a Dense"):
        alg.relational_aggregate(np.zeros((2, 2)), None, 2)
    dense = D.Dense.__new__(D.Dense)
    dense.h = None
    with pytest.raises(TypeError, match="dX must be a Dense"):
        alg.relational_aggregate_backward(dense, np.zeros(2), 2)
    with pytest.raises(RuntimeError, match="relational_aggregate failed"):
        alg.relational_aggregate(dense, dense, 2)
    with pytest.raises(RuntimeError, match="relational_aggregate_backward failed"):
        alg.relational_aggregate_backward(dense, dense, 2)
    net = D.RGCN.__new__(D.RGCN)
    net.h = None
    opt = D.AdamW()
    with pytest.raises(ValueError, match="no parameter"):
        net.param_shape(0, "neigh")
    with pytest.raises(ValueError, match="no parameter"):
        net.set_param(0, "lin", np.zeros(2))
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
    with pytest.raises(RuntimeError, match="rgcn_param_shape failed"):
        net.param_shape(0, "weight")
