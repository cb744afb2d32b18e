"""Edge softmax and softmax graph attention, CPU side: the autograd model the GPU tests compare against, and the
argument validation of the new C entry points (no GPU needed)."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import hnh_oracle as orc
from tests import gat_backward_oracle as gbo
from tests import gat_softmax_oracle as gso
from tests.mp_worker import gat_inputs


def test_edge_softmax_model_equals_dense_masked_softmax():
    """Per row, the model's edge softmax equals torch.softmax over a dense row that is -inf off the pattern."""
    N = 32
    rows, cols, _ = orc.er_tuples(5, 6, 0xC0FFEE + 9)
    ri, ci = gbo.edges(rows, cols, N)
    x = torch.from_numpy(np.random.default_rng(4).uniform(-800, 800, len(ri)))
    dense = torch.full((N, N), -torch.inf, dtype=torch.float64)
    dense[ri, ci] = x
    has = torch.isfinite(dense).any(1)
    want = torch.softmax(dense[has], 1)
    got = torch.zeros(N, N, dtype=torch.float64)
    got[ri, ci] = gso.edge_softmax_torch(x, ri, N)
    assert torch.allclose(got[has], want, rtol=1e-14, atol=1e-300)
    assert torch.isfinite(got).all()
    # the numpy restatement used by the GPU tests agrees
    assert np.allclose(gso.edge_softmax_np(x.numpy(), ri.numpy(), N), gso.edge_softmax_torch(x, ri, N).numpy(), rtol=1e-14, atol=0)


def test_edge_softmax_backward_model_equals_autograd():
    N = 16
    rows, cols, _ = orc.er_tuples(4, 5, 3)
    ri, _ = gbo.edges(rows, cols, N)
    rng = np.random.default_rng(5)
    x = torch.tensor(rng.uniform(-3, 3, len(ri)), requires_grad=True)
    g = torch.from_numpy(rng.uniform(-1, 1, len(ri)))
    a = gso.edge_softmax_torch(x, ri, N)
    a.backward(g)
    want = gso.edge_softmax_backward_np(a.detach().numpy(), g.numpy(), ri.numpy(), N)
    assert np.allclose(x.grad.numpy(), want, rtol=1e-13, atol=1e-16)


def test_softmax_gat_model_passes_gradcheck():
    """16-node graph, two layers, several heads: the autograd gradients of the softmax model equal finite
    differences."""
    N = 16
    rows, cols, _ = orc.er_tuples(4, 4, 0xC0FFEE + 5)
    ri, ci = gbo.edges(rows, cols, N)
    layers, X0, weights = gat_inputs(N, [[5, 3, 2], [6, 2, 3]], 11)
    x = torch.tensor(X0, requires_grad=True)
    ws = [torch.tensor(w, requires_grad=True) for per_layer in weights for w in per_layer]

    def f(x, *flat):
        nested, at = [], 0
        for _, _, heads in layers:
            nested.append(list(flat[at:at + heads]))
            at += heads
        return gso.gat_softmax_forward_torch(ri, ci, N, layers, nested, 0.2, x)

    assert (f(x, *ws) != 0).double().mean() > 0.2
    assert torch.autograd.gradcheck(f, (x, *ws), eps=1e-6, atol=1e-7, rtol=1e-6)


def test_softmax_gat_model_differs_from_the_leaky_one_and_is_normalised():
    N = 64
    rows, cols, _ = orc.er_tuples(6, 5, 0xC0FFEE + 3)
    layers, X0, weights = gat_inputs(N, [[12, 8, 2], [16, 4, 3]], 3)
    leaky = gbo.gat_forward_global_torch(rows, cols, N, layers, weights, 0.2, X0)
    soft = gso.gat_softmax_forward_global(rows, cols, N, layers, weights, 0.2, X0)
    assert soft.shape == leaky.shape and not np.allclose(soft, leaky)
    # one layer, one head, identity weights: each output row is a convex combination of its neighbours' rows
    ri, ci = gbo.edges(rows, cols, N)
    one = [(4, 4, 1)]
    X = np.random.default_rng(2).uniform(0.5, 1, (N, 4))
    out = gso.gat_softmax_forward_global(rows, cols, N, one, [[np.eye(4)]], 0.2, X)
    for u in np.unique(ri.numpy())[:10]:
        nb = X[ci.numpy()[ri.numpy() == u]]
        assert np.all(out[u] <= nb.max(0) + 1e-14) and np.all(out[u] >= nb.min(0) - 1e-14)


def test_edge_softmax_entry_points_validate_without_a_gpu(hnh):
    """Null pointers and negative sizes are rejected before the device is touched; empty input is a no-op."""
    buf = (C.c_double * 8)()
    p = C.addressof(buf)
    npieces = C.c_int64(-7)
    # keys
    assert hnh.hnh_edge_keys_from_index(None, None, -1, 0, None) == -1
    assert hnh.hnh_edge_keys_from_index(None, None, 0, 0, None) == 0
    assert hnh.hnh_edge_keys_from_index(p, None, 4, 0, None) == -1
    # plan
    assert hnh.hnh_edge_softmax_piece_bound(-1, 4) == -1
    assert hnh.hnh_edge_softmax_piece_bound(0, 4) == 0
    assert hnh.hnh_edge_softmax_piece_bound(3000, 2) == 2 + 3
    assert hnh.hnh_edge_softmax_piece_bound(5, 100) == 5 + 1
    assert hnh.hnh_edge_softmax_plan(p, -1, 4, p, p, p, p, 8, C.byref(npieces), None) == -1
    assert hnh.hnh_edge_softmax_plan(p, 4, -1, p, p, p, p, 8, C.byref(npieces), None) == -1
    assert hnh.hnh_edge_softmax_plan(p, 4, 1 << 31, p, p, p, p, 8, C.byref(npieces), None) == -1  # M >= 2^31
    assert b"2^31" in hnh.hnh_last_error_string()
    assert hnh.hnh_edge_softmax_plan(p, 4, 4, p, p, p, p, 8, None, None) == -1
    assert hnh.hnh_edge_softmax_plan(None, 4, 4, p, p, p, p, 8, C.byref(npieces), None) == -1
    assert hnh.hnh_edge_softmax_plan(p, 4, 4, None, p, p, p, 8, C.byref(npieces), None) == -1
    assert hnh.hnh_edge_softmax_plan(p, 4, 4, p, None, p, p, 8, C.byref(npieces), None) == -1
    # reductions and elementwise steps
    assert hnh.hnh_edge_softmax_stats_f64(p, p, p, p, p, -1, 1, p, p, p, p, None) == -1
    assert hnh.hnh_edge_softmax_stats_f64(p, p, p, p, p, 4, -1, p, p, p, p, None) == -1
    assert hnh.hnh_edge_softmax_stats_f64(None, None, None, None, None, 0, 0, None, None, None, None, None) == 0
    assert hnh.hnh_edge_softmax_stats_f64(p, p, None, p, p, 4, 2, p, p, p, p, None) == -1  # no row_start
    assert hnh.hnh_edge_softmax_stats_f64(p, p, p, p, p, 4, 2, p, p, None, p, None) == -1  # no row_max
    assert hnh.hnh_edge_softmax_stats_f64(None, p, p, p, p, 4, 2, p, p, p, p, None) == -1  # no x
    assert hnh.hnh_edge_softmax_rescale_f64(p, p, p, -1, None) == -1
    assert hnh.hnh_edge_softmax_rescale_f64(None, None, None, 0, None) == 0
    assert hnh.hnh_edge_softmax_rescale_f64(p, None, p, 4, None) == -1
    assert hnh.hnh_edge_softmax_apply_f64(p, p, p, -1, p, p, None) == -1
    assert hnh.hnh_edge_softmax_apply_f64(None, None, None, 0, None, None, None) == 0
    assert hnh.hnh_edge_softmax_apply_f64(p, p, None, 4, p, p, None) == -1
    assert hnh.hnh_edge_softmax_dot_f64(p, p, p, p, p, p, -1, 1, p, p, None) == -1
    assert hnh.hnh_edge_softmax_dot_f64(None, None, None, None, None, None, 0, 0, None, None, None) == 0
    assert hnh.hnh_edge_softmax_dot_f64(p, p, None, p, p, p, 4, 2, p, p, None) == -1  # no perm
    assert hnh.hnh_edge_softmax_dot_f64(p, p, p, p, p, p, 4, 2, p, None, None) == -1  # no row_dot
    assert hnh.hnh_edge_softmax_backward_f64(p, p, p, p, -1, p, None) == -1
    assert hnh.hnh_edge_softmax_backward_f64(None, None, None, None, 0, None, None) == 0
    assert hnh.hnh_edge_softmax_backward_f64(p, p, p, p, 4, None, None) == -1
    # driver entries: null handles
    assert hnh.hnhd_alg_edge_softmax(None, None, 0) == -1
    assert hnh.hnhd_alg_edge_softmax_backward(None, None, None, 0) == -1
    assert hnh.hnhd_gat_set_attention(None, b"softmax") == -1


def test_python_front_end_refuses_a_bogus_attention_or_order():
    from distributed_sddmm_b200 import driver as D
    with pytest.raises(ValueError, match="attention"):
        D.GAT(None, [(4, 4, 1)], attention="bogus")
    with pytest.raises(ValueError, match="mode"):
        D._value_order("C")
