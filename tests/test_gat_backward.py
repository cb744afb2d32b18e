"""GAT backward pass, CPU side: the autograd model the GPU tests compare against, and the argument validation of the
new C entry points (no GPU needed)."""
import ctypes as C

import numpy as np
import torch

from oracle import hnh_oracle as orc
from tests import gat_backward_oracle as gbo
from tests.mp_worker import gat_inputs


def test_autograd_model_passes_gradcheck():
    """16-node Erdos-Renyi graph, two layers, several heads: the autograd gradients of the model equal finite
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
        return gbo.gat_forward_torch(ri, ci, N, layers, nested, 0.2, x)

    assert (f(x, *ws) != 0).double().mean() > 0.2  # the ReLUs do not hide the attention path
    assert torch.autograd.gradcheck(f, (x, *ws), eps=1e-6, atol=1e-7, rtol=1e-6)


def test_autograd_model_forward_equals_the_numpy_model():
    N = 64
    rows, cols, _ = orc.er_tuples(6, 5, 0xC0FFEE + 3)
    layers, X0, weights = gat_inputs(N, [[12, 8, 2], [16, 4, 3]], 3)
    want = orc.gat_forward_global(rows, cols, N, layers, weights, 0.2, X0)
    have = gbo.gat_forward_global_torch(rows, cols, N, layers, weights, 0.2, X0)
    assert np.abs(have - want).max() <= 1e-14 * np.abs(want).max()


def test_backward_model_returns_every_gradient():
    N = 16
    rows, cols, _ = orc.er_tuples(4, 4, 7)
    layers, X0, weights = gat_inputs(N, [[4, 3, 2], [6, 2, 2]], 7)
    G = np.random.default_rng(1).uniform(-1, 1, (N, 4))
    dX0, dW = gbo.gat_backward_global(rows, cols, N, layers, weights, 0.2, X0, G)
    assert dX0.shape == X0.shape
    assert [[w.shape for w in per] for per in dW] == [[w.shape for w in per] for per in weights]
    # linear in the output gradient
    dX0b, dWb = gbo.gat_backward_global(rows, cols, N, layers, weights, 0.2, X0, 2 * G)
    assert np.allclose(dX0b, 2 * dX0, rtol=1e-13, atol=0) and np.allclose(dWb[1][1], 2 * dW[1][1], rtol=1e-13, atol=0)


def test_backward_entry_points_on_the_model_handle_validate_without_a_gpu(hnh):
    """Bad shapes and null pointers are rejected before the device is touched; empty sizes are successful no-ops."""
    buf = (C.c_double * 8)()
    p = C.addressof(buf)
    # TN product C (m x n) = A^T B: workspace size depends on the shape only
    assert hnh.hnh_dgemm_tn_workspace_bytes(-1, 4, 4) == -1
    assert hnh.hnh_dgemm_tn_workspace_bytes(4, 1 << 21, 4) == -1
    assert hnh.hnh_dgemm_tn_workspace_bytes(0, 4, 4) == 0 and hnh.hnh_dgemm_tn_workspace_bytes(4, 4, 0) == 0
    assert hnh.hnh_dgemm_tn_workspace_bytes(64, 64, 100) == 0  # too short a k to split
    ws = hnh.hnh_dgemm_tn_workspace_bytes(1024, 256, 1 << 20)
    assert ws > 0 and ws % (8 * 1024 * 256) == 0 and ws == hnh.hnh_dgemm_tn_workspace_bytes(1024, 256, 1 << 20)
    assert hnh.hnh_dgemm_tn_f64(None, None, None, -1, 1, 1, None, 0, None) == -1
    assert hnh.hnh_dgemm_tn_f64(None, None, None, 4, 4, -1, None, 0, None) == -1
    assert hnh.hnh_dgemm_tn_f64(None, None, None, 0, 4, 4, None, 0, None) == 0
    assert hnh.hnh_dgemm_tn_f64(None, None, None, 4, 0, 4, None, 0, None) == 0
    assert hnh.hnh_dgemm_tn_f64(None, p, p, 2, 2, 2, None, 0, None) == -1  # null C
    assert hnh.hnh_dgemm_tn_f64(p, None, p, 2, 2, 2, None, 0, None) == -1  # null A
    assert hnh.hnh_dgemm_tn_f64(p, p, p, 1024, 256, 1 << 20, None, 0, None) == -1  # no workspace
    assert b"workspace" in hnh.hnh_last_error_string()
    assert hnh.hnh_dgemm_tn_f64(p, p, p, 1024, 256, 1 << 20, p, ws - 1, None) == -1  # too small a workspace
    # NT product C (m x n) (+)= A B^T
    assert hnh.hnh_dgemm_nt_f64(None, None, None, -1, 1, 1, 0, None) == -1
    assert hnh.hnh_dgemm_nt_f64(None, None, None, 4, 4, -1, 1, None) == -1
    assert hnh.hnh_dgemm_nt_f64(None, None, None, 0, 4, 4, 0, None) == 0
    assert hnh.hnh_dgemm_nt_f64(None, None, None, 4, 0, 4, 1, None) == 0
    assert hnh.hnh_dgemm_nt_f64(None, None, None, 4, 4, 0, 1, None) == 0  # C += nothing
    assert hnh.hnh_dgemm_nt_f64(None, p, p, 2, 2, 2, 0, None) == -1
    assert hnh.hnh_dgemm_nt_f64(p, p, None, 2, 2, 2, 1, None) == -1
    # elementwise derivatives
    assert hnh.hnh_leaky_relu_grad_f64(None, None, -1, 0.2, None) == -1
    assert hnh.hnh_leaky_relu_grad_f64(None, None, 0, 0.2, None) == 0
    assert hnh.hnh_leaky_relu_grad_f64(p, None, 4, 0.2, None) == -1
    assert hnh.hnh_relu_cols_backward_f64(p, p, p, 6, 4, 2, 3, None) == -1  # window past the row end
    assert b"outside a row" in hnh.hnh_last_error_string()
    assert hnh.hnh_relu_cols_backward_f64(p, p, p, 6, 0, -1, 3, None) == -1
    assert hnh.hnh_relu_cols_backward_f64(None, None, None, 6, 2, 0, 3, None) == 0
    assert hnh.hnh_relu_cols_backward_f64(p, None, p, 6, 2, 2, 3, None) == -1
    # driver entries: null handles / pointers
    assert hnh.hnhd_model_backward(None, p) == -1
    assert hnh.hnhd_gat_get_weight_grad(None, 0, 0, p) == -1
    assert hnh.hnhd_model_get_input_grad(None, p) == -1
