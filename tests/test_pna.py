"""PNA, CPU side: the decomposed form the library computes (tests/pna_oracle.py) equals the literal per-edge PNAConv
model, both pass gradcheck away from ties and the std threshold, std is 0 with a zero gradient where it must be, the
degree averages follow PyG's formula, the numpy statistics match the torch model, and the new C and Python entry
points refuse bad arguments without a GPU."""
import ctypes as C
import itertools
import math

import numpy as np
import pytest
import torch

from tests import pna_oracle as po
from tests.test_sparse_attention_bias import _pattern

LAYERS = [(3, 4), (4, 2)]
AVG = (3.5, 1.4)
CONFIGS = [
    (("mean", "min", "max", "std"), ("identity", "amplification", "attenuation")),
    (po.AGGREGATORS, po.SCALERS),
    (("sum", "var"), ("linear", "inverse_linear")),
    (("max",), ("identity",)),
]


def _cfg(aggs, scalers):
    return (aggs, scalers) + AVG


@pytest.mark.parametrize("aggs,scalers", CONFIGS)
def test_decomposed_form_equals_the_per_edge_model(aggs, scalers):
    rng = np.random.default_rng(11)
    N = 17
    rows, cols = _pattern(rng, N, N, per_row=5)  # empty rows and a duplicate pair
    params = po.random_params(LAYERS, len(aggs), len(scalers), rng)
    tp = [{k: po._t(v) for k, v in P.items()} for P in params]
    X = po._t(rng.standard_normal((N, 3)))
    want = po.model_torch(rows, cols, N, LAYERS, tp, X, *_cfg(aggs, scalers))
    got = po.model_torch(rows, cols, N, LAYERS, tp, X, *_cfg(aggs, scalers), layer=po.layer_decomposed)
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-12)
    # and their gradients
    G = po._t(rng.standard_normal(tuple(want.shape)))
    grads = []
    for layer in (po.layer_torch, po.layer_decomposed):
        leaves = [{k: v.clone().requires_grad_() for k, v in P.items()} for P in tp]
        x = X.clone().requires_grad_()
        (po.model_torch(rows, cols, N, LAYERS, leaves, x, *_cfg(aggs, scalers), layer=layer) * G).sum().backward()
        grads.append([x.grad] + [v.grad for P in leaves for v in P.values()])
    for a, b in zip(*grads):
        assert torch.allclose(a, b, rtol=1e-10, atol=1e-10)


@pytest.mark.parametrize("aggs,scalers", CONFIGS[:3])
def test_oracle_gradcheck(aggs, scalers):
    rng = np.random.default_rng(7)
    N = 9
    rows, cols = _pattern(rng, N, N, per_row=3)
    params = po.random_params(LAYERS, len(aggs), len(scalers), rng)
    tp = [{k: po._t(v).clone().requires_grad_() for k, v in P.items()} for P in params]
    # a normal input has no ties in min / max and, on rows of two or more distinct neighbours, var far from 1e-5
    x = po._t(rng.standard_normal((N, 3))).requires_grad_()
    leaves = [x] + [v for P in tp for v in P.values()]
    names = list(tp[0])

    def f(*args):
        xx, flat = args[0], list(args[1:])
        P = [{k: flat.pop(0) for k in names} for _ in LAYERS]
        return po.model_torch(rows, cols, N, LAYERS, P, xx, *_cfg(aggs, scalers))

    assert torch.autograd.gradcheck(f, tuple(leaves), eps=1e-6, atol=1e-7)


def test_std_is_zero_with_zero_gradient_where_it_must_be():
    # row 0: three equal neighbours; row 1: one neighbour; row 2: none; row 3: two distinct neighbours
    rows, cols = np.array([0, 0, 0, 1, 3, 3]), np.array([4, 4, 4, 5, 4, 5])
    N, f = 6, 2
    x = po._t(np.random.default_rng(2).standard_normal((N, f))).requires_grad_()
    h = x[torch.as_tensor(cols)]
    out = po.aggregate_torch(h, torch.as_tensor(rows), N, "std")
    assert torch.all(out[:3] == 0) and torch.all(out[3] > 0)
    out[:3].sum().backward(retain_graph=True)
    assert torch.all(x.grad == 0)
    x.grad = None
    out[3].sum().backward()
    assert torch.all(x.grad[4:] != 0)


def test_degree_averages_follow_pyg():
    hist = np.array([2, 0, 3, 1])  # two nodes of degree 0, three of degree 2, one of degree 3
    lin, log = po.degree_averages(hist)
    assert lin == pytest.approx((2 * 3 + 3 * 1) / 6, rel=1e-15)
    assert log == pytest.approx((2 * math.log(1) + 3 * math.log(3) + math.log(4)) / 6, rel=1e-15)
    from distributed_sddmm_b200 import driver as D
    assert D.pna_degree_averages(hist) == pytest.approx((lin, log), rel=1e-15)
    for bad, match in ((np.zeros((2, 2)), "1-D"), (np.array([]), "1-D"), (np.array([1, -1]), "non-negative"),
                       (np.array([1.5]), "integer"), (np.array([0, 0]), "no node"), (np.array([np.nan]), "integer")):
        with pytest.raises(ValueError, match=match):
            D.pna_degree_averages(bad)


@pytest.mark.parametrize("which", [w for n in (1, 2, 3) for w in itertools.combinations(po.STATS, n)])
def test_numpy_statistics_match_torch(which):
    rng = np.random.default_rng(5)
    N, f = 13, 3
    rows, cols = _pattern(rng, N, N, per_row=5)
    X = rng.integers(-2, 3, (N, f)).astype(np.float64)  # ties
    A = po.multi_aggregate(rows, cols, N, X, which)
    assert A.shape == (N, po.width(which, f))
    W = po.windows(A, which, f)
    Xt = po._t(X).requires_grad_()
    r = torch.as_tensor(rows)
    h = Xt[torch.as_tensor(cols)]
    outs = {}
    if "moments" in which:
        outs["s1"] = po.aggregate_torch(h, r, N, "sum")
        outs["s2"] = po.aggregate_torch(h * h, r, N, "sum")
    for name in ("max", "min"):
        if name in which:
            outs[name] = po.aggregate_torch(h, r, N, name)
    for k, v in outs.items():
        assert np.array_equal(W[k], v.detach().numpy()), k
    dA = rng.standard_normal(A.shape)
    dW = po.windows(dA, which, f)
    sum(((v * po._t(dW[k])).sum() for k, v in outs.items())).backward()
    assert np.allclose(po.multi_aggregate_backward(rows, cols, X, A, dA, N, which), Xt.grad.numpy(), rtol=1e-13, atol=1e-13)


def test_multi_aggregate_kernels_validate_without_a_gpu(hnh):
    bufs = [(C.c_double * 256)() for _ in range(5)]
    rs, ci, x, a, d = (C.addressof(b) for b in bufs)

    def step(rs=rs, ci=ci, rows=4, nnz=4, x=x, ldx=4, f=4, which=7, a=a, lda=24):
        return hnh.hnh_multi_aggregate_step_f64(rs, ci, rows, nnz, x, ldx, f, which, a, lda, None)

    def grad(rs=rs, ci=ci, rows=4, nnz=4, x=x, ldx=4, d=d, ldd=24, f=4, which=7, dx=a, lddx=4):
        return hnh.hnh_multi_aggregate_grad_f64(rs, ci, rows, nnz, x, ldx, d, ldd, f, which, dx, lddx, None)

    for fn in (step, grad):
        assert fn(rows=-1) == -1 and b"negative" in hnh.hnh_last_error_string()
        assert fn(f=0) == -1 and b"f must be positive" in hnh.hnh_last_error_string()
        for w in (0, 8, -1):
            assert fn(which=w) == -1 and b"selects no statistic" in hnh.hnh_last_error_string()
        assert fn(f=1 << 29) == -1 and b"2^31" in hnh.hnh_last_error_string()
        assert fn(ldx=3) == -1 and b"leading dimension" in hnh.hnh_last_error_string()
        assert fn(rows=0) == 0 and fn(nnz=0, rs=None) == 0  # empty blocks are a no-op
        for k in ("rs", "ci", "x"):
            assert fn(**{k: None}) == -1 and b"null" in hnh.hnh_last_error_string(), k
    assert step(lda=23) == -1 and b"leading dimension" in hnh.hnh_last_error_string()
    assert grad(ldd=23) == -1 and grad(lddx=3) == -1
    assert step(a=x, ldx=24) == -1 and b"may not be the input" in hnh.hnh_last_error_string()
    assert grad(dx=x) == -1 and grad(dx=d, lddx=24) == -1 and b"may not be an input" in hnh.hnh_last_error_string()
    fin, prep = hnh.hnh_multi_aggregate_finish_f64, hnh.hnh_multi_aggregate_grad_prep_f64
    assert fin(a, 24, -1, 4, 7, None) == -1 and fin(a, 24, 4, 0, 7, None) == -1 and fin(a, 24, 4, 4, 0, None) == -1
    assert fin(a, 23, 4, 4, 7, None) == -1 and fin(None, 24, 4, 4, 7, None) == -1
    assert fin(None, 8, 4, 4, 1, None) == 0  # moments only: nothing to finish
    assert prep(a, 24, d, 24, 4, 4, 7, a, 24, None) == -1 and b"may not be an input" in hnh.hnh_last_error_string()
    assert prep(a, 24, d, 23, 4, 4, 7, x, 24, None) == -1 and prep(a, 24, d, 24, 4, 4, 9, x, 24, None) == -1
    comb, cgrad = hnh.hnh_pna_combine_f64, hnh.hnh_pna_combine_grad_f64
    # four aggregators (codes 0, 2, 3, 5), three scalers (0, 1, 2): P is 13 f wide
    assert comb(x, 4, x, 4, a, 24, 7, d, 1, 4, 4, 0x5320, 4, 0x210, 3, 1.0, 1.0, a, 51, None) == -1
    assert b"leading dimension" in hnh.hnh_last_error_string()
    assert comb(x, 4, x, 4, a, 24, 7, d, 1, 4, 4, 0x5326, 4, 0x210, 3, 1.0, 1.0, a, 52, None) == -1
    assert b"unknown code" in hnh.hnh_last_error_string()
    assert comb(x, 4, x, 4, a, 24, 7, d, 1, 4, 4, 0x5320, 0, 0x210, 3, 1.0, 1.0, a, 52, None) == -1
    assert comb(x, 4, x, 4, a, 24, 7, d, 1, 4, 4, 0x5320, 4, 0x510, 3, 1.0, 1.0, a, 52, None) == -1
    assert comb(None, 4, x, 4, a, 24, 7, d, 1, 4, 4, 0x5320, 4, 0x210, 3, 1.0, 1.0, a, 52, None) == -1
    # an aggregator whose statistic the state does not hold: min and max without their windows, mean without moments
    for aggs, which in ((0x5320, 1), (0x5320, 3), (0x5320, 5), (0x0, 6)):
        assert comb(x, 4, x, 4, a, 24, which, d, 1, 4, 4, aggs, 4 if aggs else 1, 0x210, 3, 1.0, 1.0, a, 52, None) == -1
        assert b"does not hold" in hnh.hnh_last_error_string()
        assert cgrad(a, 52, a, 24, which, d, 1, 4, 4, aggs, 4 if aggs else 1, 0x210, 3, 1.0, 1.0, x, 4, d, 24, None) == -1
        assert b"does not hold" in hnh.hnh_last_error_string()
    assert cgrad(a, 51, a, 24, 7, d, 1, 4, 4, 0x5320, 4, 0x210, 3, 1.0, 1.0, x, 4, d, 24, None) == -1
    assert cgrad(a, 52, a, 24, 7, None, 1, 4, 4, 0x5320, 4, 0x210, 3, 1.0, 1.0, x, 4, d, 24, None) == -1
    if not torch.cuda.is_available():  # no CPU fallback: compute fails with HNH_E_CUDA
        assert step() == -2 and grad() == -2 and fin(a, 24, 4, 4, 7, None) == -2


def test_pna_create_and_aggregation_validate_without_a_gpu(hnh):
    out = C.c_void_p()
    res = (C.c_double * 4)()
    p = C.addressof(res)
    layers = (C.c_int * 4)(3, 4, 4, 2)
    a, s = b"mean,max", b"identity"
    assert hnh.hnhd_pna_create(None, 2, layers, a, s, 1.0, 1.0, C.byref(out)) == -1 and b"bad argument" in hnh.hnh_last_error_string()
    assert hnh.hnhd_pna_create(p, 0, layers, a, s, 1.0, 1.0, C.byref(out)) == -1
    assert hnh.hnhd_pna_create(p, 2, None, a, s, 1.0, 1.0, C.byref(out)) == -1
    assert hnh.hnhd_pna_create(p, 2, layers, None, s, 1.0, 1.0, C.byref(out)) == -1
    assert hnh.hnhd_pna_create(p, 2, layers, a, None, 1.0, 1.0, C.byref(out)) == -1
    assert hnh.hnhd_pna_create(p, 2, layers, a, s, 1.0, 1.0, None) == -1
    for bad in (np.zeros((2, 2)), [1, -1], [0, 0]):  # a given histogram is checked even where no scaler reads it
        from distributed_sddmm_b200 import driver as D
        alg = D.Algorithm.__new__(D.Algorithm)
        alg.h = None
        with pytest.raises(ValueError, match="deg"):
            D.PNA(alg, [(3, 4)], scalers=("identity",), deg=bad)
    with pytest.raises(ValueError, match="needed by the scalers"):
        D.PNA(alg, [(3, 4)], scalers=("identity", "linear"))
    for args in ((None, p, p), (p, None, p), (p, p, None)):
        assert hnh.hnhd_alg_multi_aggregate(*args, 7) == -1 and b"null" in hnh.hnh_last_error_string()
        assert hnh.hnhd_alg_multi_aggregate_backward(*args, p, p, 7, 0) == -1 and b"null" in hnh.hnh_last_error_string()


def test_python_front_end_validates_pna_arguments():
    from distributed_sddmm_b200 import driver as D
    alg = D.Algorithm.__new__(D.Algorithm)
    alg.h = None
    with pytest.raises(ValueError, match="pairs"):
        D.PNA(alg, [(3, 4, 2)], deg=[1, 2])
    with pytest.raises(ValueError, match="pairs"):
        D.PNA(alg, [], deg=[1, 2])
    with pytest.raises(RuntimeError, match="pna_create failed"):
        D.PNA(alg, [(3, 4)], deg=[1, 2])  # null algorithm handle
    for which in ((), ("moments", "moments"), ("mean",), "sum"):
        with pytest.raises(ValueError, match="which"):
            alg.multi_aggregate(None, None, which)
    assert D.Algorithm.multi_aggregate_width(("moments", "min"), 5) == 20
    with pytest.raises(TypeError, match="X must be a Dense"):
        alg.multi_aggregate(np.zeros((2, 2)), None)
    dense = D.Dense.__new__(D.Dense)
    dense.h = None
    with pytest.raises(TypeError, match="dX must be a Dense"):
        alg.multi_aggregate_backward(dense, dense, dense, np.zeros(2))
    with pytest.raises(RuntimeError, match="multi_aggregate failed"):
        alg.multi_aggregate(dense, dense)
    with pytest.raises(RuntimeError, match="multi_aggregate_backward failed"):
        alg.multi_aggregate_backward(dense, dense, dense, dense)
    net = D.PNA.__new__(D.PNA)
    net.h = None
    with pytest.raises(RuntimeError, match="pna_param_shape failed"):
        net.param_shape(0, "pre")
    assert net.param_names() == ["pre", "pre_bias", "post", "post_bias", "lin", "lin_bias"]
