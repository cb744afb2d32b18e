"""R-GCN with basis decomposition, CPU side: the fp64 oracle (tests/rgcn_basis_oracle.py) against finite differences for
both aggregators including comp, against the per-relation oracle when the bases are the relations, the numpy kernels
against the torch model (H, dX and dcomp, with and without the mean's scale, with values that are no relation), and
the new C and Python entry points refuse bad arguments without a GPU."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import rgcn_basis_oracle as bo
from tests import rgcn_oracle as ro
from tests.test_sparse_attention_bias import _pattern

LAYERS = [(3, 4), (4, 2)]


@pytest.mark.parametrize("aggr", bo.AGGREGATIONS)
def test_oracle_gradcheck(aggr):
    rng = np.random.default_rng(11)
    N, R, B = 9, 3, 2
    rows, cols = _pattern(rng, N, N, per_row=3)
    rows, cols = np.append(rows, [2, 2]), np.append(cols, [5, 5])  # a duplicate pair
    rels = rng.integers(0, R, len(rows)).astype(np.float64)
    rels[-2:] = [0, 2]  # ... under two relations
    params = bo.random_params(LAYERS, R, B, rng)
    tp = [{k: bo._t(v).clone().requires_grad_() for k, v in P.items()} for P in params]
    x = bo._t(rng.standard_normal((N, 3))).requires_grad_()
    leaves = [x] + [v for P in tp for v in P.values()]
    names = list(params[0])

    def f(*args):
        xx, flat = args[0], list(args[1:])
        P = [{k: flat.pop(0) for k in names} for _ in LAYERS]
        return bo.model_torch(rows, cols, rels, N, LAYERS, P, xx, R, B, aggr)

    assert torch.autograd.gradcheck(f, tuple(leaves), eps=1e-6, atol=1e-7)


@pytest.mark.parametrize("aggr", bo.AGGREGATIONS)
def test_identity_bases_are_the_relations(aggr):
    """B = R and comp = I: the basis model is the per-relation model with weight = basis, gradients included."""
    rng = np.random.default_rng(4)
    N, R = 12, 3
    rows, cols = _pattern(rng, N, N, per_row=4)
    rels = rng.integers(0, R, len(rows)).astype(np.float64)
    params = bo.random_params(LAYERS, R, R, rng)
    for P in params:
        P["comp"] = np.eye(R)
    X, G = rng.standard_normal((N, 3)), rng.standard_normal((N, 2))
    out, dX, dP = bo.forward_backward(rows, cols, rels, N, LAYERS, params, X, R, R, aggr, G)
    plain = [{k: P[k] for k in ro.PARAMS} for P in params]
    out2, dX2, dP2 = ro.forward_backward(rows, cols, rels, N, LAYERS, plain, X, R, aggr, G)
    assert np.allclose(out, out2, rtol=1e-14, atol=1e-14) and np.allclose(dX, dX2, rtol=1e-13, atol=1e-13)
    for g, g2 in zip(dP, dP2):
        for k in ro.PARAMS:
            assert np.allclose(g[k], g2[k], rtol=1e-13, atol=1e-13), k


@pytest.mark.parametrize("mean", [False, True])
def test_numpy_kernels_match_the_torch_model(mean):
    """H, dX and dcomp of the numpy kernels against autograd of the basis-first sums; values that are no relation
    (-1, R, 0.5, NaN, +-inf) count nowhere."""
    rng = np.random.default_rng(5 + mean)
    N, R, B, f = 13, 4, 3, 3
    rows, cols = _pattern(rng, N, N, per_row=5)
    rels = rng.integers(0, R, len(rows)).astype(np.float64)
    rels[::7] = np.resize([-1.0, R, 0.5, np.nan, np.inf, -np.inf], len(rels[::7]))
    scale = bo.mean_scale(rows, rels, N, R) if mean else None
    X = bo._t(rng.standard_normal((N, f))).requires_grad_()
    comp = bo._t(rng.standard_normal((R, B))).requires_grad_()
    dH = rng.standard_normal((N, B * f))
    ok = ro.valid(rels, R)
    rel = np.where(ok, np.nan_to_num(rels), 0).astype(np.int64)
    w = np.ones(len(rows)) if scale is None else scale[rows, rel]
    # H as a torch sum over the entries, entry by entry
    H = torch.zeros(N, B, f, dtype=torch.float64)
    for j in np.flatnonzero(ok):
        H[rows[j]] = H[rows[j]] + w[j] * comp[rel[j]][:, None] * X[cols[j]][None, :]
    want = bo.basis_aggregate(rows, cols, rels, N, X.detach().numpy(), R, comp.detach().numpy(), scale)
    assert np.allclose(H.reshape(N, B * f).detach().numpy(), want, rtol=1e-13, atol=1e-13)
    (H.reshape(N, B * f) * bo._t(dH)).sum().backward()
    dX, dcomp = bo.basis_aggregate_backward(rows, cols, rels, dH, X.detach().numpy(), N, R, comp.detach().numpy(), scale)
    assert np.allclose(dX, X.grad.numpy(), rtol=1e-13, atol=1e-13)
    assert np.allclose(dcomp, comp.grad.numpy(), rtol=1e-13, atol=1e-13)
    # the per-entry products sum to dcomp by relation (B order: the stored row is X's, the gathered one dH's)
    P = bo.products(rows, cols, rels, dH, X.detach().numpy(), R, B, scale)
    assert not P[:, ~ok].any()
    by_rel = np.zeros((R, B))
    np.add.at(by_rel, rel[ok], P[:, ok].T)
    assert np.allclose(by_rel, dcomp, rtol=1e-13, atol=1e-13)


def test_mean_scale_is_the_inverse_count():
    rows, rels = np.array([0, 0, 0, 1, 1]), np.array([0.0, 1.0, 1.0, 0.0, 0.5])
    assert np.array_equal(bo.mean_scale(rows, rels, 3, 2), [[1.0, 0.5], [1.0, 0.0], [0.0, 0.0]])


def test_basis_kernels_validate_without_a_gpu(hnh):
    bufs = [(C.c_double * 64)() for _ in range(8)]
    rs, ci, v, x, h, cp, sc, pp = (C.addressof(b) for b in bufs)

    def agg(rs=rs, ci=ci, v=v, rows=4, nnz=4, x=x, ldx=4, f=4, s=None, lds=0, cp=cp, R=2, B=2, h=h, ldh=8):
        return hnh.hnh_basis_aggregate_f64(rs, ci, v, rows, nnz, x, ldx, f, s, lds, cp, R, B, h, ldh, None)

    def grad(rs=rs, ci=ci, v=v, rows=4, nnz=4, dh=h, lddh=8, s=None, lds=0, cp=cp, R=2, B=2, x=x, ldx=4, f=4, dx=sc, lddx=4,
             p=None, ldp=4):
        return hnh.hnh_basis_aggregate_grad_f64(rs, ci, v, rows, nnz, dh, lddh, s, lds, cp, R, B, x, ldx, f, dx, lddx, p, ldp, None)

    for fn in (agg, grad):
        assert fn(rows=-1) == -1 and b"negative" in hnh.hnh_last_error_string()
        assert fn(f=0) == -1 and b"f must be positive" in hnh.hnh_last_error_string()
        assert fn(R=0) == -1 and b"relation count" in hnh.hnh_last_error_string()
        assert fn(B=0) == -1 and b"basis count" in hnh.hnh_last_error_string()
        assert fn(B=1 << 20, f=1 << 12) == -1 and b"below 2^31" in hnh.hnh_last_error_string()
        assert fn(R=1 << 20, B=1 << 12) == -1 and b"below 2^31" in hnh.hnh_last_error_string()
        assert fn(s=sc if fn is agg else h, lds=1) == -1 and b"leading dimension" in hnh.hnh_last_error_string()
        assert fn(rows=0) == 0 and fn(nnz=0, rs=None) == 0  # empty blocks are a no-op
        for k in ("rs", "ci", "v", "cp"):
            assert fn(**{k: None}) == -1 and b"null" in hnh.hnh_last_error_string(), k
    for kw in (dict(ldx=3), dict(ldh=7)):
        assert agg(**kw) == -1 and b"leading dimension" in hnh.hnh_last_error_string(), kw
    for kw in (dict(lddh=7), dict(lddx=3), dict(p=pp, ldx=3), dict(p=pp, ldp=3)):
        assert grad(**kw) == -1 and b"leading dimension" in hnh.hnh_last_error_string(), kw
    assert agg(x=None) == -1 and agg(h=None) == -1 and grad(dh=None) == -1 and grad(dx=None) == -1
    assert grad(p=pp, x=None) == -1 and b"null" in hnh.hnh_last_error_string()
    for kw in (dict(h=x, ldh=8, ldx=8), dict(h=v), dict(h=cp), dict(h=sc, s=sc, lds=2)):
        assert agg(**kw) == -1 and b"may not be an input" in hnh.hnh_last_error_string(), kw
    for kw in (dict(dx=h, lddx=8), dict(dx=v), dict(dx=cp), dict(p=h), dict(p=pp, dx=pp), dict(p=pp, x=pp)):
        assert grad(**kw) == -1 and b"may not be" in hnh.hnh_last_error_string(), kw
    rk = hnh.hnh_relation_keys
    assert rk(pp, v, -1, 2, None) == -1 and rk(pp, v, 4, 0, None) == -1
    assert rk(None, v, 4, 2, None) == -1 and rk(pp, None, 4, 2, None) == -1 and rk(None, None, 0, 2, None) == 0
    if not torch.cuda.is_available():  # no CPU fallback: compute fails with HNH_E_CUDA
        assert agg() == -2 and grad() == -2 and grad(p=pp) == -2 and rk(pp, v, 4, 2, None) == -2


def test_basis_driver_entry_points_validate_without_a_gpu(hnh):
    out = C.c_void_p()
    res = (C.c_double * 4)()
    p = C.addressof(res)
    layers = (C.c_int * 4)(3, 4, 4, 2)
    create = hnh.hnhd_rgcn_create_bases
    assert create(None, 2, layers, 3, 2, b"mean", C.byref(out)) == -1 and b"bad argument" in hnh.hnh_last_error_string()
    assert create(p, 0, layers, 3, 2, b"mean", C.byref(out)) == -1
    assert create(p, 2, None, 3, 2, b"mean", C.byref(out)) == -1
    assert create(p, 2, layers, 3, 2, None, C.byref(out)) == -1
    assert create(p, 2, layers, 3, 2, b"mean", None) == -1
    # refused before the algorithm is touched
    for nb in (0, -1):
        assert create(p, 2, layers, 3, nb, b"mean", C.byref(out)) == -1 and b"basis count" in hnh.hnh_last_error_string()
    assert create(p, 2, layers, 0, 2, b"mean", C.byref(out)) == -1 and b"relation count" in hnh.hnh_last_error_string()
    assert create(p, 2, layers, 3, 2, b"max", C.byref(out)) == -1 and b"unknown aggregation" in hnh.hnh_last_error_string()
    bad = (C.c_int * 4)(3, 4, 5, 2)
    assert create(p, 2, bad, 3, 2, b"sum", C.byref(out)) == -1 and b"does not take the width" in hnh.hnh_last_error_string()
    wide = (C.c_int * 2)(1 << 20, 4)
    assert create(p, 1, wide, 3, 1 << 12, b"sum", C.byref(out)) == -1 and b"B f must be below 2^31" in hnh.hnh_last_error_string()
    assert create(p, 1, layers, 1 << 20, 1 << 12, b"sum", C.byref(out)) == -1 and b"R B must be below" in hnh.hnh_last_error_string()
    for args in ((None, p, p, p), (p, None, p, p), (p, p, None, p), (p, p, p, None)):
        assert hnh.hnhd_alg_basis_aggregate(*args, 2, None) == -1 and b"null" in hnh.hnh_last_error_string()
    for i in range(6):
        args = [p] * 6
        args[i] = None
        assert hnh.hnhd_alg_basis_aggregate_backward(*args[:5], args[5], 2, None, 0) == -1
        assert b"null" in hnh.hnh_last_error_string()


def test_python_front_end_validates_basis_arguments():
    from distributed_sddmm_b200 import driver as D
    alg = D.Algorithm.__new__(D.Algorithm)
    alg.h = None
    for nb in (0, -2):
        with pytest.raises(ValueError, match="num_bases"):
            D.RGCN(alg, [(3, 4)], num_relations=2, num_bases=nb)
    with pytest.raises(ValueError, match="aggr"):
        D.RGCN(alg, [(3, 4)], num_relations=2, aggr="max", num_bases=2)
    with pytest.raises(RuntimeError, match="rgcn_create_bases failed"):
        D.RGCN(alg, [(3, 4)], num_relations=2, num_bases=2)  # null algorithm handle
    with pytest.raises(TypeError, match="X must be a Dense"):
        alg.basis_aggregate(np.zeros((2, 2)), None, np.eye(2), 2)
    dense = D.Dense.__new__(D.Dense)
    dense.h = None
    with pytest.raises(TypeError, match="H must be a Dense"):
        alg.basis_aggregate(dense, np.zeros(2), np.eye(2), 2)
    with pytest.raises(TypeError, match="scale must be a Dense"):
        alg.basis_aggregate(dense, dense, np.eye(2), 2, scale=np.ones((2, 2)))
    with pytest.raises(TypeError, match="dX must be a Dense"):
        alg.basis_aggregate_backward(dense, dense, np.zeros(2), np.eye(2), 2)
    for comp in (np.zeros(3), np.zeros((2, 0)), np.zeros((2, 2, 2))):
        with pytest.raises(ValueError, match="comp must be an R x B matrix"):
            alg.basis_aggregate(dense, dense, comp, 2)
        with pytest.raises(ValueError, match="comp must be an R x B matrix"):
            alg.basis_aggregate_backward(dense, dense, dense, comp, 2)
    net = D.RGCN.__new__(D.RGCN)
    net.h = None
    net.num_bases = 3
    assert net.param_names() == ["weight", "comp", "bias", "root"]
    with pytest.raises(ValueError, match="no parameter"):
        net.param_shape(0, "basis")
    with pytest.raises(RuntimeError, match="rgcn_param_shape failed"):
        net.param_shape(0, "comp")
    net.num_bases = None
    with pytest.raises(ValueError, match="no parameter"):
        net.param_shape(0, "comp")  # no comp without bases
