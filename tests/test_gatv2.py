"""GATv2 attention, CPU side: the autograd model the GPU tests compare against (checked with gradcheck and against a
dense masked-softmax restatement), its difference from additive attention, and the argument validation of the new C
entry points (no GPU needed)."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import hnh_oracle as orc
from tests import gat_additive_oracle as gao
from tests import gatv2_oracle as g2
from tests.mp_worker import gat_inputs


def test_gatv2_model_passes_gradcheck():
    """16-node graph, two layers, several heads: the autograd gradients of X0, every W and every a equal finite
    differences."""
    N = 16
    rows, cols, _ = orc.er_tuples(4, 4, 0xC0FFEE + 5)
    ri, ci = g2.edges(rows, cols, N)
    layers, X0, weights = gat_inputs(N, [[5, 3, 2], [6, 2, 3]], 11)
    a = g2.attention_inputs(layers, 11)
    x = torch.tensor(X0, requires_grad=True)
    flat = [torch.tensor(v, requires_grad=True) for nested in (weights, a) for per_layer in nested for v in per_layer]
    per = sum(heads for _, _, heads in layers)

    def nest(vs):
        out, at = [], 0
        for _, _, heads in layers:
            out.append(list(vs[at:at + heads]))
            at += heads
        return out

    def f(x, *flat):
        return g2.gatv2_forward_torch(ri, ci, N, layers, nest(flat[:per]), nest(flat[per:]), 0.2, x)

    assert (f(x, *flat) != 0).double().mean() > 0.2
    assert torch.autograd.gradcheck(f, (x, *flat), eps=1e-6, atol=1e-7, rtol=1e-6)


def test_gatv2_model_equals_dense_masked_softmax():
    """The edge-list model equals an N x N masked torch.softmax formulation, and both LeakyReLU branches occur."""
    N = 64
    rows, cols, _ = orc.er_tuples(6, 5, 0xC0FFEE + 3)
    ri, ci = g2.edges(rows, cols, N)
    layers, X0, weights = gat_inputs(N, [[12, 8, 2], [16, 5, 3]], 3)
    a = g2.attention_inputs(layers, 3)
    t = lambda nested: [[torch.from_numpy(v) for v in per_layer] for per_layer in nested]  # noqa: E731
    args = (ri, ci, N, layers, t(weights), t(a), 0.2, torch.from_numpy(X0))
    got = g2.gatv2_forward_torch(*args)
    want = g2.gatv2_forward_dense(*args)
    assert torch.abs(want).max() > 0
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-14)
    H = torch.from_numpy(X0) @ torch.from_numpy(weights[0][0])
    z = H[ri] + H[ci]
    assert (z > 0).any() and (z < 0).any()
    # the kernel-level numpy references agree with the model's score
    Hn = H.numpy()
    x = g2.scores_np(Hn, Hn, ri.numpy(), ci.numpy(), a[0][0], 0.2)
    assert np.allclose(x, (torch.nn.functional.leaky_relu(z, 0.2) @ torch.from_numpy(a[0][0])).numpy(), rtol=1e-14, atol=1e-15)


def test_gatv2_is_dynamic_and_zero_vectors_give_mean_aggregation():
    """Unlike additive attention, GATv2 lets different nodes rank the same neighbours differently; with a = 0 both
    are the mean over each node's neighbours."""
    N = 32
    rows, cols, _ = orc.er_tuples(5, 6, 7)
    layers, X0, weights = gat_inputs(N, [[6, 4, 1]], 7)
    H = X0 @ weights[0][0]
    a = np.array([1.0, -1.0, 0.5, 2.0])
    # two nodes u1, u2 and two candidate neighbours v1, v2: the preferred neighbour depends on u
    score = lambda u, v: g2.scores_np(H, H, np.array([u]), np.array([v]), a, 0.2)[0]  # noqa: E731
    flips = [(u1, u2, v1, v2) for u1 in range(8) for u2 in range(8) for v1 in range(8) for v2 in range(8)
             if (score(u1, v1) - score(u1, v2)) * (score(u2, v1) - score(u2, v2)) < 0]
    assert flips
    zeros = [[np.zeros(fph) for _ in range(heads)] for _, fph, heads in layers]
    v2 = g2.gatv2_forward_global(rows, cols, N, layers, weights, zeros, 0.2, X0)
    add = gao.gat_additive_forward_global(rows, cols, N, layers, weights, zeros, zeros, 0.2, X0)
    assert np.allclose(v2, add, rtol=1e-14, atol=1e-15)
    nonzero = g2.gatv2_forward_global(rows, cols, N, layers, weights, g2.attention_inputs(layers, 7), 0.2, X0)
    assert not np.allclose(nonzero, v2)


def test_gatv2_entry_points_validate_without_a_gpu(hnh):
    """Null pointers, negative sizes, r < 1 and leading dimensions below r are rejected before the device is touched;
    empty input is a no-op."""
    buf = (C.c_double * 8)()
    p = C.addressof(buf)

    def scores(rs=p, ci=p, rows=4, nnz=4, R=p, ldr=4, Y=p, ldy=4, a=p, r=4, out=p):
        return hnh.hnh_gatv2_scores_f64(rs, ci, rows, nnz, R, ldr, Y, ldy, a, r, 0.2, out, None)

    def grad(rs=p, ci=p, g=p, rows=4, nnz=4, R=p, ldr=4, Y=p, ldy=4, a=p, r=4, dR=p, lddr=4, da=None, ws=None, wsb=0):
        return hnh.hnh_gatv2_grad_f64(rs, ci, g, rows, nnz, R, ldr, Y, ldy, a, r, 0.2, dR, lddr, da, ws, wsb, None)

    for call in (scores, grad):
        assert call(rows=-1) == -1
        assert call(nnz=-1) == -1
        assert call(r=0) == -1
        assert b"r must be positive" in hnh.hnh_last_error_string()
        assert call(ldr=3) == -1
        assert b"leading dimension" in hnh.hnh_last_error_string()
        assert call(ldy=3) == -1
        assert call(rs=None) == -1
        assert b"null pointer" in hnh.hnh_last_error_string()
        assert call(ci=None) == -1
        assert call(R=None) == -1
        assert call(Y=None) == -1
        assert call(a=None) == -1
        # empty blocks: nothing to do, nothing touched
        assert call(rs=None, ci=None, R=None, Y=None, a=None, rows=0) == 0
        assert call(rs=None, ci=None, R=None, Y=None, a=None, nnz=0) == 0
    assert scores(out=None) == -1
    assert grad(g=None) == -1
    assert grad(dR=None) == -1
    assert grad(lddr=3) == -1
    assert b"dR" in hnh.hnh_last_error_string()
    # da needs a workspace of hnh_gatv2_grad_workspace_bytes(rows, r) bytes
    assert grad(da=p) == -1
    assert b"workspace" in hnh.hnh_last_error_string()
    need = hnh.hnh_gatv2_grad_workspace_bytes(4, 4)
    assert need == 4 * 4 * 8
    assert grad(da=p, ws=p, wsb=need - 1) == -1
    assert hnh.hnh_gatv2_grad_workspace_bytes(-1, 4) == -1
    assert hnh.hnh_gatv2_grad_workspace_bytes(4, 0) == -1
    assert hnh.hnh_gatv2_grad_workspace_bytes(0, 4) == 0
    assert hnh.hnh_gatv2_grad_workspace_bytes(1 << 30, 256) == hnh.hnh_gatv2_grad_workspace_bytes(1 << 20, 256) > 0
    # driver entries: null handles and arguments, bad value orders
    assert hnh.hnhd_alg_gatv2_scores(None, p, p, p, p, 0, 0.2) == -1
    assert hnh.hnhd_alg_gatv2_backward(None, p, p, p, p, p, p, p, p, 0.2) == -1
    assert b"null argument" in hnh.hnh_last_error_string()
    assert hnh.hnhd_gat_set_attention(None, b"gatv2") == -1


def test_python_front_end_refuses_a_misspelt_kind_and_a_bad_value_order():
    """The Python front end refuses "GATv2", naming every kind, and value orders other than "A" and "B"."""
    from distributed_sddmm_b200 import driver as D
    assert "gatv2" in D.GAT.ATTENTIONS
    with pytest.raises(ValueError, match="additive.*gatv2"):
        D.GAT(None, [(4, 4, 1)], attention="GATv2")
    with pytest.raises(ValueError, match='mode must be "A" or "B"'):
        D._value_order("C")
