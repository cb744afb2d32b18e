"""GIN and GINE, CPU side: the literal per-edge oracle (tests/gin_oracle.py) equals a plain nn.Module pipeline with
PyG's GINConv / GINEConv state-dict layout, the oracle passes gradcheck away from the ReLUs' kinks, the numpy
edge-ReLU aggregation matches it, and the new C and Python entry points refuse bad arguments without a GPU."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import gin_oracle as go
from tests.test_sparse_attention_bias import _pattern

LAYERS = [(3, 5, 4), (4, 6, 2)]


class _GINEConv(torch.nn.Module):
    """GINConv (edge_dim 0) or GINEConv as PyG writes them: nn((1 + eps) x + sum_j msg_j), msg_j = x_j or
    relu(x_j + lin(edge_attr)), aggregated by a scatter-add over the target."""

    def __init__(self, f, h, r, edge_dim):
        super().__init__()
        self.nn = torch.nn.Sequential(torch.nn.Linear(f, h), torch.nn.ReLU(), torch.nn.Linear(h, r)).double()
        self.lin = torch.nn.Linear(edge_dim, f).double() if edge_dim else None
        self.eps = torch.nn.Parameter(torch.zeros(1, dtype=torch.float64))

    def forward(self, x, edge_index, edge_attr=None):
        src, dst = edge_index
        msg = x[src] if self.lin is None else torch.relu(x[src] + self.lin(edge_attr))
        out = torch.zeros_like(x).scatter_add_(0, dst[:, None].expand(-1, x.shape[1]), msg)
        return self.nn((1 + self.eps) * x + out)


def _load(conv, P):
    """The library's parameters -> a GINConv / GINEConv state dict (weights transposed)."""
    sd = {"nn.0.weight": P["lin1"].T, "nn.0.bias": P["lin1_bias"], "nn.2.weight": P["lin2"].T, "nn.2.bias": P["lin2_bias"],
          "eps": P["eps"]}
    if "edge" in P:
        sd.update({"lin.weight": P["edge"].T, "lin.bias": P["edge_bias"]})
    conv.load_state_dict({k: go._t(v) for k, v in sd.items()})


@pytest.mark.parametrize("edge_dim", [0, 3])
def test_oracle_equals_an_nn_module_pipeline(edge_dim):
    rng = np.random.default_rng(5)
    N = 17
    rows, cols = _pattern(rng, N, N, per_row=5)  # empty rows and a duplicate pair
    params = go.random_params(LAYERS, edge_dim, rng)
    attr = go._t(go.attr_of(rows, cols, edge_dim)) if edge_dim else None
    X = go._t(rng.standard_normal((N, 3)))
    convs = []
    for (f, h, r), P in zip(LAYERS, params):
        conv = _GINEConv(f, h, r, edge_dim)
        _load(conv, P)
        convs.append(conv)
    ei = torch.as_tensor(np.stack([cols, rows]).astype(np.int64))
    h = X
    for l, conv in enumerate(convs):
        h = conv(h, ei, attr)
        h = torch.relu(h) if l + 1 < len(convs) else h
    tp = [{k: go._t(v) for k, v in P.items()} for P in params]
    want = go.model_torch(rows, cols, N, LAYERS, tp, X, attr)
    assert torch.allclose(h, want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("edge_dim", [0, 2])
def test_oracle_gradcheck(edge_dim):
    rng = np.random.default_rng(7)
    N = 9
    rows, cols = _pattern(rng, N, N, per_row=3)
    params = go.random_params(LAYERS, edge_dim, rng)
    tp = [{k: go._t(v).clone().requires_grad_() for k, v in P.items()} for P in params]
    attr = go._t(go.attr_of(rows, cols, edge_dim)) if edge_dim else None
    X = go._t(rng.standard_normal((N, 3))).requires_grad_()
    leaves = [X] + [v for P in tp for v in P.values()]
    # normal inputs keep every ReLU argument away from 0, where its derivative jumps
    assert torch.autograd.gradcheck(lambda *_: go.model_torch(rows, cols, N, LAYERS, tp, X, attr), leaves, eps=1e-6, atol=1e-7)


def test_numpy_edge_relu_aggregation_matches_torch():
    rng = np.random.default_rng(3)
    N, f = 13, 4
    rows, cols = _pattern(rng, N, N, per_row=4)
    X = rng.integers(-2, 3, (N, f)).astype(np.float64)
    E = rng.integers(-2, 3, (len(rows), f)).astype(np.float64)  # X_v + E_i == 0 happens: the strict mask
    assert (X[cols] + E == 0).any()
    Xt, Et = go._t(X).requires_grad_(), go._t(E).requires_grad_()
    A = torch.zeros(N, f, dtype=torch.float64).index_add_(0, torch.as_tensor(rows), torch.relu(Xt[torch.as_tensor(cols)] + Et))
    assert np.array_equal(go.edge_relu_aggregate(rows, cols, N, X, E), A.detach().numpy())
    dA = rng.standard_normal((N, f))
    (A * go._t(dA)).sum().backward()
    dX, dE = go.edge_relu_aggregate_backward(rows, cols, X, E, dA, N)
    assert np.allclose(dX, Xt.grad.numpy(), rtol=1e-13, atol=1e-13) and np.array_equal(dE, Et.grad.numpy())


def test_edge_relu_kernels_validate_without_a_gpu(hnh):
    bufs = [(C.c_double * 256)() for _ in range(6)]
    rs, ci, x, e, a, d = (C.addressof(b) for b in bufs)

    def step(rs=rs, ci=ci, rows=4, nnz=4, x=x, ldx=4, e=e, lde=4, f=4, a=a, lda=4):
        return hnh.hnh_edge_relu_aggregate_step_f64(rs, ci, rows, nnz, x, ldx, e, lde, f, a, lda, None)

    def grad(rs=rs, ci=ci, rows=4, nnz=4, x=x, ldx=4, e=e, lde=4, a=d, lda=4, f=4, dx=a, lddx=4):
        return hnh.hnh_edge_relu_aggregate_grad_f64(rs, ci, rows, nnz, x, ldx, e, lde, a, lda, f, dx, lddx, None)

    def egrad(rs=rs, ci=ci, rows=4, nnz=4, a=d, lda=4, x=x, ldx=4, e=e, lde=4, f=4, de=a, ldde=4):
        return hnh.hnh_edge_relu_aggregate_edge_grad_f64(rs, ci, rows, nnz, a, lda, x, ldx, e, lde, f, de, ldde, None)

    for fn in (step, grad, egrad):
        assert fn(rows=-1) == -1 and b"negative" in hnh.hnh_last_error_string()
        assert fn(f=0) == -1 and b"f must be positive" in hnh.hnh_last_error_string()
        for ld in ("ldx", "lde", "lda"):
            assert fn(**{ld: 3}) == -1 and b"leading dimension" in hnh.hnh_last_error_string(), (fn, ld)
        assert fn(rows=0) == 0 and fn(nnz=0, rs=None) == 0  # empty blocks are a no-op
        for k in ("rs", "ci", "x", "e"):
            assert fn(**{k: None}) == -1 and b"null" in hnh.hnh_last_error_string(), k
    assert step(a=None) == -1 and grad(a=None) == -1 and grad(dx=None) == -1 and egrad(de=None) == -1
    assert grad(lddx=3) == -1 and egrad(ldde=3) == -1
    assert step(a=x) == -1 and step(a=e) == -1 and b"may not be an input" in hnh.hnh_last_error_string()
    for alias in (x, e, d):
        assert grad(dx=alias) == -1 and b"may not be an input" in hnh.hnh_last_error_string()
    assert egrad(de=x) == -1 and egrad(de=e) == -1 and egrad(de=d) == -1
    comb, cgrad = hnh.hnh_gin_combine_f64, hnh.hnh_gin_combine_grad_f64
    assert comb(a, d, x, e, -1, None) == -1 and comb(a, d, x, None, 4, None) == -1 and comb(x, d, x, e, 4, None) == -1
    assert comb(None, d, x, e, 0, None) == 0
    assert cgrad(a, None, d, x, e, -1, None) == -1 and cgrad(a, None, d, x, None, 4, None) == -1
    assert cgrad(d, None, d, x, e, 4, None) == -1 and cgrad(a, e, d, None, e, 4, None) == -1
    if not torch.cuda.is_available():  # no CPU fallback: compute fails with HNH_E_CUDA
        assert step() == -2 and grad() == -2 and egrad() == -2 and comb(a, d, x, e, 4, None) == -2


def test_gin_create_and_aggregation_validate_without_a_gpu(hnh):
    out = C.c_void_p()
    res = (C.c_double * 4)()
    p = C.addressof(res)
    layers = (C.c_int * 6)(3, 5, 4, 4, 6, 2)
    assert hnh.hnhd_gin_create(None, 2, layers, 0, 0.0, 0, C.byref(out)) == -1 and b"bad argument" in hnh.hnh_last_error_string()
    assert hnh.hnhd_gin_create(p, 0, layers, 0, 0.0, 0, C.byref(out)) == -1
    assert hnh.hnhd_gin_create(p, 2, None, 0, 0.0, 0, C.byref(out)) == -1
    assert hnh.hnhd_gin_create(p, 2, layers, 0, 0.0, 0, None) == -1
    assert hnh.hnhd_gin_set_edge_attributes(None, p, 1, p, 1) == -1 and b"null model" in hnh.hnh_last_error_string()
    for args in ((None, p, p, p), (p, None, p, p), (p, p, None, p), (p, p, p, None)):
        assert hnh.hnhd_alg_edge_relu_aggregate(*args) == -1 and b"null" in hnh.hnh_last_error_string()
    for args in ((None, p, p, p, p), (p, None, p, p, p), (p, p, p, None, p), (p, p, p, p, None)):
        X, EA, dA, dX = args[1], args[2], args[3], args[4]
        assert hnh.hnhd_alg_edge_relu_aggregate_backward(args[0], X, EA, EA, dA, dX, None, 0) == -1
        assert b"null" in hnh.hnh_last_error_string()


def test_python_front_end_validates_gin_arguments():
    from distributed_sddmm_b200 import driver as D
    alg = D.Algorithm.__new__(D.Algorithm)
    alg.h = None
    for layers in ([(3, 4)], [], [(3, 4, 2, 1)]):
        with pytest.raises(ValueError, match="triples"):
            D.GIN(alg, layers)
    with pytest.raises(ValueError, match="chain"):
        D.GIN(alg, [(3, 4, 2), (3, 4, 2)])
    for edge_dim in (-1, 1.5, True):
        with pytest.raises(ValueError, match="edge_dim"):
            D.GIN(alg, [(3, 4, 2)], edge_dim=edge_dim)
    for eps in (float("nan"), float("inf"), "0", True):
        with pytest.raises(ValueError, match="eps"):
            D.GIN(alg, [(3, 4, 2)], eps=eps)
    with pytest.raises(RuntimeError, match="gin_create failed"):
        D.GIN(alg, [(3, 4, 2)])  # null algorithm handle
    with pytest.raises(TypeError, match="E must be a Dense"):
        alg.edge_relu_aggregate(None, np.zeros((2, 2)), None)
    dense = D.Dense.__new__(D.Dense)
    dense.h = None
    with pytest.raises(TypeError, match="dE must be a Dense"):
        alg.edge_relu_aggregate_backward(dense, dense, dense, dense, dense, np.zeros(2))
    with pytest.raises(RuntimeError, match="edge_relu_aggregate failed"):
        alg.edge_relu_aggregate(dense, dense, dense)
    with pytest.raises(RuntimeError, match="edge_relu_aggregate_backward failed"):
        alg.edge_relu_aggregate_backward(dense, dense, dense, dense, dense)
    net = D.GIN.__new__(D.GIN)
    net.h, net.edge_dim = None, 0
    with pytest.raises(RuntimeError, match="gin_param_shape failed"):
        net.param_shape(0, "lin1")
    with pytest.raises(ValueError, match="no edge features"):
        net.set_edge_attributes(np.zeros((2, 1)), np.zeros((2, 1)))
    assert net.param_names() == ["lin1", "lin1_bias", "lin2", "lin2_bias", "eps"]
    net.edge_dim = 2
    assert net.param_names() == ["lin1", "lin1_bias", "lin2", "lin2_bias", "edge", "edge_bias", "eps"]
    with pytest.raises(ValueError, match="attr_B must be n x 2"):
        net.set_edge_attributes(np.zeros((2, 2)), np.zeros((2, 3)))
    with pytest.raises(RuntimeError, match="gin_set_edge_attributes failed"):
        net.set_edge_attributes(np.zeros((2, 2)), np.zeros((2, 2)))
