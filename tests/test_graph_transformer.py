"""Graph transformer, CPU side: the fp64 model the GPU tests compare against (gradcheck in every parameter, in X and in
the edge attributes for all four (gate, edge) combinations; with W_e = 0 and no gate it is the sparse attention model
composed with the projections), and the argument validation of the new C entry points, driver entries and Python
front end (no GPU needed)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from tests import graph_transformer_oracle as gto
from tests import sparse_attention_oracle as sa
from tests.test_sparse_attention_bias import _pattern

LAYERS = [(3, 2, 2), (4, 3, 1)]


def _square_pattern(rng, N):
    rows, cols = _pattern(rng, N, N, per_row=3)  # empty rows and a duplicate pair
    return rows, cols


@pytest.mark.parametrize("beta", [False, True])
@pytest.mark.parametrize("edge_dim", [0, 2])
def test_model_passes_gradcheck(beta, edge_dim):
    rng = np.random.default_rng(11 + edge_dim + beta)
    N = 7
    rows, cols = _square_pattern(rng, N)
    params = gto.random_params(LAYERS, edge_dim, beta, rng, scale=0.8)
    names = [sorted(P) for P in params]
    flat = [torch.tensor(params[l][n], requires_grad=True) for l in range(len(LAYERS)) for n in names[l]]
    X = torch.tensor(rng.standard_normal((N, LAYERS[0][0])), requires_grad=True)
    args = [X] + flat
    if edge_dim:
        args.append(torch.tensor(gto.dense_attributes(rows, cols, N, rng.standard_normal((len(rows), edge_dim))),
                                 requires_grad=True))
    p = 0.3 if beta else 0.0

    def f(x, *rest):
        it = iter(rest)
        P = [{n: next(it) for n in names[l]} for l in range(len(LAYERS))]
        A = next(it) if edge_dim else None
        return gto.model_torch(rows, cols, N, LAYERS, P, x, A, beta, p, 5)

    assert torch.autograd.gradcheck(f, args, eps=1e-6, atol=1e-8, rtol=1e-6)


def test_model_without_edge_and_gate_is_projected_sparse_attention():
    """W_e = 0 and no gate: every layer is ReLU(sparse_attention(X W_q + b_q, X W_k + b_k, X W_v + b_v) + X W_s + b_s)
    with the sparse attention oracle's per-entry formulation (and no ReLU after the last)."""
    rng = np.random.default_rng(29)
    N = 23
    rows, cols = _square_pattern(rng, N)
    layers = [(5, 3, 2), (6, 2, 3), (6, 4, 1)]
    params = gto.random_params(layers, 3, False, rng)
    for P in params:
        P["edge"][:] = 0.0
    X = rng.standard_normal((N, 5))
    attr = rng.standard_normal((len(rows), 3))
    got = gto.forward_np(rows, cols, N, layers, params, X, attr)
    x = X
    for l, (f, d, H) in enumerate(layers):
        P = params[l]
        Q, K, V, R = (x @ P[n] + P[n + "_bias"] for n in gto.PROJECTIONS)
        Z, _ = sa.forward_np(rows, cols, N, Q, K, V, H, 1 / math.sqrt(d))
        x = Z + R
        if l + 1 < len(layers):
            x = np.maximum(x, 0.0)
    assert np.allclose(got, x, rtol=1e-13, atol=1e-13)
    assert np.abs(x).max() > 0


def test_gate_backward_formulas():
    """dM, dR and dw_beta of the issue's closed form equal autograd's on one gated combine."""
    rng = np.random.default_rng(3)
    n, r = 9, 5
    M, R, dY = (torch.tensor(rng.standard_normal((n, r)), requires_grad=True) for _ in range(3))
    w = torch.tensor(rng.standard_normal(3 * r), requires_grad=True)
    b = torch.sigmoid(torch.cat([M, R, M - R], 1) @ w)[:, None]
    (b * R + (1 - b) * M).backward(dY.detach())
    with torch.no_grad():
        ds = ((dY * (R - M)).sum(1, keepdim=True)) * b * (1 - b)
        w1, w2, w3 = w[:r], w[r:2 * r], w[2 * r:]
        assert torch.allclose(M.grad, (1 - b) * dY + ds * (w1 + w3), rtol=1e-14, atol=1e-14)
        assert torch.allclose(R.grad, b * dY + ds * (w2 - w3), rtol=1e-14, atol=1e-14)
        assert torch.allclose(w.grad, (ds * torch.cat([M, R, M - R], 1)).sum(0), rtol=1e-13, atol=1e-13)


def test_kernel_entry_points_validate_without_a_gpu(hnh):
    """Negative sizes, null pointers, aliasing outputs, a gate without dw_beta (and the reverse) and a short workspace
    are refused before the device is touched; empty sizes are successful no-ops; a real call fails cleanly without a
    device."""
    bufs = [(C.c_double * 64)() for _ in range(8)]
    a, b, c, d, e, f, g, h = (C.addressof(x) for x in bufs)
    assert hnh.hnh_row_bias_add_f64(a, b, -1, 4, None) == -1 and b"negative" in hnh.hnh_last_error_string()
    assert hnh.hnh_row_bias_add_f64(a, b, 4, -1, None) == -1
    assert hnh.hnh_row_bias_add_f64(None, b, 4, 4, None) == -1 and b"null" in hnh.hnh_last_error_string()
    assert hnh.hnh_row_bias_add_f64(a, None, 4, 4, None) == -1
    assert hnh.hnh_row_bias_add_f64(None, None, 0, 4, None) == 0 and hnh.hnh_row_bias_add_f64(None, None, 4, 0, None) == 0

    assert hnh.hnh_gt_gate_f64(a, b, c, None, -1, 4, 0, None) == -1
    assert hnh.hnh_gt_gate_f64(None, b, c, d, 4, 4, 1, None) == -1 and b"null" in hnh.hnh_last_error_string()
    assert hnh.hnh_gt_gate_f64(a, None, c, None, 4, 4, 1, None) == -1
    assert hnh.hnh_gt_gate_f64(a, b, None, None, 4, 4, 1, None) == -1
    assert hnh.hnh_gt_gate_f64(b, b, c, None, 4, 4, 1, None) == -1 and b"Y may not be" in hnh.hnh_last_error_string()
    assert hnh.hnh_gt_gate_f64(c, b, c, d, 4, 4, 1, None) == -1
    assert hnh.hnh_gt_gate_f64(None, None, None, None, 0, 4, 1, None) == 0

    ws = hnh.hnh_gt_gate_backward_workspace_bytes(1000, 7)
    assert ws >= 8 * (1000 + 3 * 7) and ws == hnh.hnh_gt_gate_backward_workspace_bytes(1000, 7)
    assert hnh.hnh_gt_gate_backward_workspace_bytes(-1, 7) == -1

    def bw(dM=a, dR=b, dw=c, G=d, Y=e, M=f, R=g, w=h, n=4, r=4, relu=1, ws_p=a, ws_bytes=1 << 20):
        return hnh.hnh_gt_gate_backward_f64(dM, dR, dw, G, Y, M, R, w, n, r, relu, ws_p, ws_bytes, None)

    assert bw(n=-1) == -1 and bw(r=-1) == -1
    assert bw(dw=None) == -1 and b"needs dw_beta" in hnh.hnh_last_error_string()
    assert bw(w=None) == -1 and b"dw_beta without the gate" in hnh.hnh_last_error_string()
    assert bw(dM=None) == -1 and bw(G=None) == -1 and bw(M=None) == -1 and bw(R=None) == -1
    assert bw(Y=None) == -1 and b"null" in hnh.hnh_last_error_string()
    assert bw(dR=None) == -1  # the gate writes dR
    assert bw(dM=d) == -1 and b"may not be an input" in hnh.hnh_last_error_string()
    assert bw(dR=g) == -1 and bw(dw=h) == -1
    assert bw(dR=a) == -1 and b"one matrix" in hnh.hnh_last_error_string()
    assert bw(ws_p=None) == -1 and b"workspace" in hnh.hnh_last_error_string()
    need = hnh.hnh_gt_gate_backward_workspace_bytes(4, 4)
    assert bw(ws_bytes=need - 1) == -1
    assert bw(r=0) == 0 and bw(w=None, dw=None, r=0) == 0 and bw(w=None, dw=None, n=0) == 0
    if not torch.cuda.is_available():
        assert hnh.hnh_row_bias_add_f64(a, b, 4, 4, None) == -2
        assert hnh.hnh_gt_gate_f64(a, b, c, d, 4, 4, 1, None) == -2
        assert bw(ws_bytes=need) == -2
        assert bw(w=None, dw=None, dR=None, Y=None, relu=0) == -2


def test_driver_entry_points_validate_without_a_gpu(hnh):
    """Null handles and arguments are refused by every hnhd_gt_* entry point."""
    buf = (C.c_double * 8)()
    p = C.addressof(buf)
    i64 = C.c_int64()
    layers = (C.c_int * 3)(4, 2, 2)
    out = C.c_void_p()
    assert hnh.hnhd_gt_create(None, 1, layers, 0, 0, C.byref(out)) == -1
    assert hnh.hnhd_gt_create(p, 0, layers, 0, 0, C.byref(out)) == -1
    assert hnh.hnhd_gt_create(p, 1, None, 0, 0, C.byref(out)) == -1
    assert hnh.hnhd_gt_create(p, 1, layers, 0, 0, None) == -1
    assert b"bad argument" in hnh.hnh_last_error_string()
    for name in (b"query", b"beta", b"nope"):
        assert hnh.hnhd_gt_param_shape(None, 0, name, C.byref(i64), C.byref(i64)) == -1
        assert hnh.hnhd_gt_set_param(None, 0, name, p) == -1
        assert hnh.hnhd_gt_get_param(None, 0, name, p) == -1
        assert hnh.hnhd_gt_get_param_grad(None, 0, name, p) == -1
    assert hnh.hnhd_gt_buffer_shape(None, 0, C.byref(i64), C.byref(i64)) == -1
    assert hnh.hnhd_gt_set_input(None, p) == -1
    assert hnh.hnhd_gt_get_buffer(None, 0, p) == -1
    assert hnh.hnhd_gt_set_edge_attributes(None, p, 1, p, 1) == -1
    assert hnh.hnhd_gt_forward(None, 0.0, 0) == -1
    assert hnh.hnhd_gt_backward(None, p) == -1
    assert hnh.hnhd_gt_get_input_grad(None, p) == -1
    assert b"null" in hnh.hnh_last_error_string()
    hnh.hnhd_gt_destroy(None)  # a no-op


def test_python_front_end_validates_arguments():
    """The front end refuses these before it touches the handle (here a null one)."""
    from distributed_sddmm_b200 import driver as D
    alg = D.Algorithm.__new__(D.Algorithm)
    alg.h = None
    for bad in (-1, 1.5, True, "2"):
        with pytest.raises(ValueError, match="edge_dim"):
            D.GraphTransformer(alg, [(4, 2, 2)], edge_dim=bad)
    with pytest.raises(ValueError, match="triples"):
        D.GraphTransformer(alg, [(4, 2)])
    with pytest.raises(RuntimeError, match="gt_create failed"):
        D.GraphTransformer(alg, [(4, 2, 2)])  # null algorithm handle
    gt = D.GraphTransformer.__new__(D.GraphTransformer)
    gt.h, gt.layers, gt.edge_dim, gt.beta = None, [(4, 2, 2)], 0, False
    assert gt.param_names() == ["query", "query_bias", "key", "key_bias", "value", "value_bias", "skip", "skip_bias"]
    gt.edge_dim, gt.beta = 3, True
    assert gt.param_names()[-2:] == ["edge", "beta"]
    for bad in (-0.1, 1.0, math.nan):
        with pytest.raises(ValueError, match="dropout"):
            gt.forward(dropout=bad)
    for bad in (-1, 1 << 64, 0.5, True):
        with pytest.raises(ValueError, match="seed"):
            gt.forward(seed=bad)
    with pytest.raises(ValueError, match="n x 3"):
        gt.set_edge_attributes(np.zeros((4, 2)), np.zeros((4, 3)))
    with pytest.raises(ValueError, match="n x 3"):
        gt.set_edge_attributes(np.zeros((4, 3)), np.zeros(4))
    gt.edge_dim = 0
    with pytest.raises(ValueError, match="no edge features"):
        gt.set_edge_attributes(np.zeros((4, 3)), np.zeros((4, 3)))
    gt.h = None
