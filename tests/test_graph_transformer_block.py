"""Graph transformer blocks, CPU side: the fp64 model the GPU tests compare against (gradcheck in every parameter, in X
and in the edge attributes, with and without the gate; with a zero feed-forward network a layer is LN2(LN1(Y))), the
LayerNorm backward's closed form, and the argument validation of the new C entry points, driver entry and Python front
end (no GPU needed)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import graph_transformer_block_oracle as gbo
from tests import graph_transformer_oracle as gto
from tests.test_sparse_attention_bias import _pattern

LAYERS = [(3, 2, 2), (4, 3, 1)]


@pytest.mark.parametrize("beta", [False, True])
@pytest.mark.parametrize("edge_dim", [0, 2])
def test_block_model_passes_gradcheck(beta, edge_dim):
    rng = np.random.default_rng(41 + edge_dim + beta)
    N = 7
    rows, cols = _pattern(rng, N, N, per_row=3)
    ffn = 2 if beta else 1
    params = gbo.random_params(LAYERS, edge_dim, beta, ffn, rng, scale=0.8)
    names = [sorted(P) for P in params]
    flat = [torch.tensor(params[l][n], requires_grad=True) for l in range(len(LAYERS)) for n in names[l]]
    X = torch.tensor(rng.standard_normal((N, LAYERS[0][0])), requires_grad=True)
    args = [X] + flat
    if edge_dim:
        args.append(torch.tensor(gto.dense_attributes(rows, cols, N, rng.standard_normal((len(rows), edge_dim))),
                                 requires_grad=True))
    p = 0.3 if edge_dim else 0.0

    def f(x, *rest):
        it = iter(rest)
        P = [{n: next(it) for n in names[l]} for l in range(len(LAYERS))]
        A = next(it) if edge_dim else None
        return gbo.model_torch(rows, cols, N, LAYERS, P, x, A, beta, p, 5, eps=1e-3)

    assert torch.autograd.gradcheck(f, args, eps=1e-6, atol=1e-8, rtol=1e-6)


@pytest.mark.parametrize("beta", [False, True])
def test_zero_ffn_is_two_layer_norms(beta):
    """With the FFN's weights and biases zero every layer is LN2(LN1(Y)), Y the TransformerConv output of
    tests/graph_transformer_oracle.py before its ReLU."""
    rng = np.random.default_rng(7 + beta)
    N = 23
    rows, cols = _pattern(rng, N, N, per_row=3)
    layers = [(5, 3, 2), (6, 2, 3)]
    params = gbo.random_params(layers, 2, beta, 2, rng)
    for P in params:
        P["ffn1"][:] = 0.0
        P["ffn2"][:] = 0.0
    X = rng.standard_normal((N, 5))
    attr = rng.standard_normal((len(rows), 2))
    got = gbo.forward_np(rows, cols, N, layers, params, X, attr, beta, 0.3, 9)
    x, s = X, 9
    for l, lay in enumerate(layers):
        Y = gto.forward_np(rows, cols, N, [lay], [params[l]], x, attr, beta, 0.3, s)
        r = Y.shape[1]
        ln = lambda v, g, b: F.layer_norm(torch.from_numpy(v), (r,), torch.from_numpy(g), torch.from_numpy(b), 1e-5).numpy()
        x = ln(ln(Y, params[l]["norm1"], params[l]["norm1_bias"]), params[l]["norm2"], params[l]["norm2_bias"])
        s += lay[2]
    assert np.allclose(got, x, rtol=1e-13, atol=1e-13)
    assert np.abs(x).max() > 0


def test_layer_norm_backward_formulas():
    """dU, dgamma and dbeta of the closed form equal autograd's on one LayerNorm of X + Res."""
    rng = np.random.default_rng(5)
    n, r, eps = 9, 6, 1e-5
    X, Res, G = (torch.tensor(rng.standard_normal((n, r)), requires_grad=True) for _ in range(3))
    g, b = (torch.tensor(rng.standard_normal(r), requires_grad=True) for _ in range(2))
    F.layer_norm(X + Res, (r,), g, b, eps).backward(G.detach())
    with torch.no_grad():
        x = X + Res
        mean = x.mean(1, keepdim=True)
        rstd = 1 / torch.sqrt(((x - mean) ** 2).mean(1, keepdim=True) + eps)
        xh = (x - mean) * rstd
        gg = G * g
        dU = rstd * (gg - gg.mean(1, keepdim=True) - xh * (gg * xh).mean(1, keepdim=True))
        assert torch.allclose(X.grad, dU, rtol=1e-13, atol=1e-13) and torch.allclose(Res.grad, dU, rtol=1e-13, atol=1e-13)
        assert torch.allclose(g.grad, (G * xh).sum(0), rtol=1e-13, atol=1e-13)
        assert torch.allclose(b.grad, G.sum(0), rtol=1e-13, atol=1e-13)


def test_block_kernel_entry_points_validate_without_a_gpu(hnh):
    """Negative sizes, a bad eps, null pointers, aliasing outputs and a short workspace are refused before the device
    is touched; empty sizes are successful no-ops; a real call fails cleanly without a device."""
    bufs = [(C.c_double * 64)() for _ in range(9)]
    a, b, c, d, e, f, g, h, w = (C.addressof(x) for x in bufs)
    assert hnh.hnh_row_bias_relu_f64(a, b, c, -1, 4, None) == -1 and b"negative" in hnh.hnh_last_error_string()
    assert hnh.hnh_row_bias_relu_f64(a, b, c, 4, -1, None) == -1
    for args in ((None, b, c), (a, None, c), (a, b, None)):
        assert hnh.hnh_row_bias_relu_f64(*args, 4, 4, None) == -1 and b"null" in hnh.hnh_last_error_string()
    assert hnh.hnh_row_bias_relu_f64(b, b, c, 4, 4, None) == -1 and b"may not be" in hnh.hnh_last_error_string()
    assert hnh.hnh_row_bias_relu_f64(c, b, c, 4, 4, None) == -1
    assert hnh.hnh_row_bias_relu_f64(None, None, None, 0, 4, None) == 0
    assert hnh.hnh_row_bias_relu_f64(None, None, None, 4, 0, None) == 0

    def fw(Y=a, st=b, X=c, Res=d, gm=e, bt=f, n=4, r=4, eps=1e-5):
        return hnh.hnh_layer_norm_f64(Y, st, X, Res, gm, bt, n, r, eps, None)

    assert fw(n=-1) == -1 and b"negative" in hnh.hnh_last_error_string()
    assert fw(r=-1) == -1
    for bad in (0.0, -1e-5, math.nan, math.inf, -math.inf):
        assert fw(eps=bad) == -1 and b"eps" in hnh.hnh_last_error_string()
        assert fw(n=0, eps=bad) == -1
    for k in ("Y", "st", "X", "gm", "bt"):
        assert fw(**{k: None}) == -1 and b"null" in hnh.hnh_last_error_string(), k
    for out in ("Y", "st"):
        for src in (c, d, e, f):
            assert fw(**{out: src}) == -1 and b"may not be an input" in hnh.hnh_last_error_string()
    assert fw(st=a) == -1 and b"one buffer" in hnh.hnh_last_error_string()
    assert fw(n=0, Y=None, st=None, X=None, gm=None, bt=None) == 0 and fw(r=0) == 0

    ws = hnh.hnh_layer_norm_backward_workspace_bytes(1000, 7)
    assert ws >= 8 * 2 * 7 and ws == hnh.hnh_layer_norm_backward_workspace_bytes(1000, 7)
    assert hnh.hnh_layer_norm_backward_workspace_bytes(-1, 7) == -1
    assert hnh.hnh_layer_norm_backward_workspace_bytes(7, -1) == -1

    def bw(dX=a, dg=b, db=c, G=d, X=e, Res=f, st=g, gm=h, n=4, r=4, acc=0, ws_p=w, ws_bytes=1 << 20):
        return hnh.hnh_layer_norm_backward_f64(dX, dg, db, G, X, Res, st, gm, n, r, acc, ws_p, ws_bytes, None)

    assert bw(n=-1) == -1 and b"negative" in hnh.hnh_last_error_string()
    assert bw(r=-1) == -1
    for k in ("dX", "dg", "db", "G", "X", "st", "gm"):
        assert bw(**{k: None}) == -1 and b"null" in hnh.hnh_last_error_string(), k
    for out in ("dX", "dg", "db"):
        for src in (d, e, f, g, h):
            assert bw(**{out: src}) == -1 and b"may not be an input" in hnh.hnh_last_error_string()
    assert bw(db=b) == -1 and b"one vector" in hnh.hnh_last_error_string()
    assert bw(dX=b) == -1 and b"one buffer" in hnh.hnh_last_error_string()
    assert bw(ws_p=None) == -1 and b"workspace" in hnh.hnh_last_error_string()
    need = hnh.hnh_layer_norm_backward_workspace_bytes(4, 4)
    assert bw(ws_bytes=need - 1) == -1
    assert bw(r=0) == 0 and bw(r=0, dX=None, G=None, X=None, st=None, gm=None, ws_p=None) == 0
    if not torch.cuda.is_available():
        assert hnh.hnh_row_bias_relu_f64(a, b, c, 4, 4, None) == -2
        assert fw() == -2 and fw(Res=None) == -2
        assert bw(ws_bytes=need) == -2
        assert bw(n=0) == -2  # the zero fill of dgamma and dbeta needs the device


def test_block_driver_entry_point_validates_without_a_gpu(hnh):
    buf = (C.c_double * 8)()
    p = C.addressof(buf)
    layers = (C.c_int * 3)(4, 2, 2)
    out = C.c_void_p()
    assert hnh.hnhd_gt_create_block(None, 1, layers, 0, 0, 1, 1e-5, C.byref(out)) == -1
    assert hnh.hnhd_gt_create_block(p, 0, layers, 0, 0, 1, 1e-5, C.byref(out)) == -1
    assert hnh.hnhd_gt_create_block(p, 1, None, 0, 0, 1, 1e-5, C.byref(out)) == -1
    assert hnh.hnhd_gt_create_block(p, 1, layers, 0, 0, 1, 1e-5, None) == -1
    assert b"bad argument" in hnh.hnh_last_error_string()
    i64 = C.c_int64()
    for name in (b"norm1", b"norm1_bias", b"ffn1", b"ffn2", b"norm2", b"norm2_bias"):
        assert hnh.hnhd_gt_param_shape(None, 0, name, C.byref(i64), C.byref(i64)) == -1
        assert hnh.hnhd_gt_set_param(None, 0, name, p) == -1
        assert hnh.hnhd_gt_get_param_grad(None, 0, name, p) == -1


def test_python_front_end_validates_block_arguments():
    from distributed_sddmm_b200 import driver as D
    alg = D.Algorithm.__new__(D.Algorithm)
    alg.h = None
    for bad in (-1, 1.5, True, "2", None):
        with pytest.raises(ValueError, match="ffn_ratio"):
            D.GraphTransformer(alg, [(4, 2, 2)], ffn_ratio=bad)
    for bad in (0.0, -1e-5, math.nan, math.inf, "1e-5", True, None):
        with pytest.raises(ValueError, match="norm_eps"):
            D.GraphTransformer(alg, [(4, 2, 2)], ffn_ratio=1, norm_eps=bad)
    with pytest.raises(ValueError, match="triples"):
        D.GraphTransformer(alg, [(4, 2)], ffn_ratio=2)
    with pytest.raises(RuntimeError, match="gt_create_block failed"):
        D.GraphTransformer(alg, [(4, 2, 2)], ffn_ratio=2)  # null algorithm handle
    with pytest.raises(RuntimeError, match="gt_create failed"):
        D.GraphTransformer(alg, [(4, 2, 2)], ffn_ratio=0)
    gt = D.GraphTransformer.__new__(D.GraphTransformer)
    gt.h, gt.layers, gt.edge_dim, gt.beta = None, [(4, 2, 2)], 3, True
    base = ["query", "query_bias", "key", "key_bias", "value", "value_bias", "skip", "skip_bias", "edge", "beta"]
    assert gt.param_names() == base  # an object without the option reads it as 0
    gt.ffn_ratio = 0
    assert gt.param_names() == base
    gt.ffn_ratio = 2
    assert gt.param_names() == base + ["norm1", "norm1_bias", "ffn1", "ffn2", "norm2", "norm2_bias"]
    gt.h = None
