"""Additive graph attention, CPU side: the autograd model the GPU tests compare against (checked with gradcheck and
against a dense masked-softmax restatement), and the argument validation of the new C entry points (no GPU needed)."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import hnh_oracle as orc
from tests import gat_additive_oracle as gao
from tests import gat_softmax_oracle as gso
from tests.mp_worker import gat_inputs


def test_additive_gat_model_passes_gradcheck():
    """16-node graph, two layers, several heads: the autograd gradients of X0, every W, a1 and a2 equal finite
    differences."""
    N = 16
    rows, cols, _ = orc.er_tuples(4, 4, 0xC0FFEE + 5)
    ri, ci = gao.edges(rows, cols, N)
    layers, X0, weights = gat_inputs(N, [[5, 3, 2], [6, 2, 3]], 11)
    a1, a2 = gao.attention_inputs(layers, 11)
    x = torch.tensor(X0, requires_grad=True)
    flat = [torch.tensor(v, requires_grad=True) for nested in (weights, a1, a2) for per_layer in nested for v in per_layer]
    per = sum(heads for _, _, heads in layers)

    def nest(vs):
        out, at = [], 0
        for _, _, heads in layers:
            out.append(list(vs[at:at + heads]))
            at += heads
        return out

    def f(x, *flat):
        return gao.gat_additive_forward_torch(ri, ci, N, layers, nest(flat[:per]), nest(flat[per:2 * per]),
                                              nest(flat[2 * per:]), 0.2, x)

    assert (f(x, *flat) != 0).double().mean() > 0.2
    assert torch.autograd.gradcheck(f, (x, *flat), eps=1e-6, atol=1e-7, rtol=1e-6)


def test_additive_gat_model_equals_dense_masked_softmax():
    """The edge-list model equals an N x N masked torch.softmax formulation, and both LeakyReLU branches occur."""
    N = 64
    rows, cols, _ = orc.er_tuples(6, 5, 0xC0FFEE + 3)
    ri, ci = gao.edges(rows, cols, N)
    layers, X0, weights = gat_inputs(N, [[12, 8, 2], [16, 4, 3]], 3)
    a1, a2 = gao.attention_inputs(layers, 3)
    t = lambda nested: [[torch.from_numpy(v) for v in per_layer] for per_layer in nested]  # noqa: E731
    args = (ri, ci, N, layers, t(weights), t(a1), t(a2), 0.2, torch.from_numpy(X0))
    got = gao.gat_additive_forward_torch(*args)
    want = gao.gat_additive_forward_dense(*args)
    assert torch.abs(want).max() > 0
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-14)
    # the first head's scores take both signs
    H = torch.from_numpy(X0) @ torch.from_numpy(weights[0][0])
    x = (H @ torch.from_numpy(a1[0][0]))[ri] + (H @ torch.from_numpy(a2[0][0]))[ci]
    assert (x > 0).any() and (x < 0).any()
    # zero attention vectors: uniform attention, i.e. the mean over each node's neighbours
    z = [[np.zeros(fph) for _ in range(heads)] for _, fph, heads in layers]
    one = [(12, 8, 1)]
    mean = gao.gat_additive_forward_global(rows, cols, N, one, [weights[0][:1]], z[:1], z[:1], 0.2, X0)
    H = X0 @ weights[0][0]
    ri_np, ci_np = ri.numpy(), ci.numpy()
    for u in np.unique(ri_np)[:10]:
        assert np.allclose(mean[u], np.maximum(H[ci_np[ri_np == u]].mean(0), 0), rtol=1e-13, atol=1e-15)


def test_additive_gat_differs_from_softmax_attention():
    N = 32
    rows, cols, _ = orc.er_tuples(5, 5, 7)
    layers, X0, weights = gat_inputs(N, [[6, 4, 2]], 7)
    a1, a2 = gao.attention_inputs(layers, 7)
    add = gao.gat_additive_forward_global(rows, cols, N, layers, weights, a1, a2, 0.2, X0)
    soft = gso.gat_softmax_forward_global(rows, cols, N, layers, weights, 0.2, X0)
    assert add.shape == soft.shape and not np.allclose(add, soft)


def test_additive_entry_points_validate_without_a_gpu(hnh):
    """Null pointers and negative sizes are rejected before the device is touched; empty input is a no-op."""
    buf = (C.c_double * 8)()
    p = C.addressof(buf)
    # node scalars s = P a1, t = P a2
    assert hnh.hnh_gat_node_scalars_f64(p, p, p, p, p, -1, 4, None) == -1
    assert hnh.hnh_gat_node_scalars_f64(p, p, p, p, p, 4, -1, None) == -1
    assert hnh.hnh_gat_node_scalars_f64(None, None, None, None, None, 0, 4, None) == 0
    assert hnh.hnh_gat_node_scalars_f64(None, p, p, p, p, 4, 4, None) == -1  # no s
    assert hnh.hnh_gat_node_scalars_f64(p, p, None, p, p, 4, 4, None) == -1  # no P
    assert hnh.hnh_gat_node_scalars_f64(p, p, p, p, None, 4, 4, None) == -1  # no a2
    # edge scores
    assert hnh.hnh_gat_edge_scores_f64(p, p, p, p, p, -1, 0.2, 0, None) == -1
    assert hnh.hnh_gat_edge_scores_f64(None, None, None, None, None, 0, 0.2, 1, None) == 0
    assert hnh.hnh_gat_edge_scores_f64(p, p, p, p, None, 4, 0.2, 0, None) == -1  # no column keys
    assert hnh.hnh_gat_edge_scores_f64(p, None, p, p, p, 4, 0.2, 1, None) == -1  # no s
    # rank-2 row update
    assert hnh.hnh_gat_rank2_update_f64(p, p, p, p, p, -1, 4, None) == -1
    assert hnh.hnh_gat_rank2_update_f64(p, p, p, p, p, 4, -1, None) == -1
    assert hnh.hnh_gat_rank2_update_f64(None, None, None, None, None, 0, 4, None) == 0
    assert hnh.hnh_gat_rank2_update_f64(None, None, None, None, None, 4, 0, None) == 0
    assert hnh.hnh_gat_rank2_update_f64(p, p, None, p, p, 4, 4, None) == -1  # no dt
    # row / column sums over a plan
    assert hnh.hnh_edge_sum_f64(p, p, p, p, p, -1, 1, p, p, None) == -1
    assert hnh.hnh_edge_sum_f64(p, p, p, p, p, 4, -1, p, p, None) == -1
    assert hnh.hnh_edge_sum_f64(None, None, None, None, None, 0, 0, None, None, None) == 0
    assert hnh.hnh_edge_sum_f64(p, None, p, p, p, 4, 2, p, p, None) == -1  # no perm
    assert hnh.hnh_edge_sum_f64(p, p, p, p, p, 4, 2, p, None, None) == -1  # no row_sum
    assert hnh.hnh_edge_sum_f64(None, p, p, p, p, 4, 2, p, p, None) == -1  # no x
    # driver entries: null handles and pointers
    assert hnh.hnhd_gat_set_attention(None, b"additive") == -1
    assert hnh.hnhd_gat_set_attention_vectors(None, 0, 0, p, p) == -1
    assert hnh.hnhd_gat_set_attention_vectors(None, 0, 0, None, p) == -1
    assert hnh.hnhd_gat_get_attention_grads(None, 0, 0, p, p) == -1
    assert hnh.hnhd_gat_get_attention_grads(None, 0, 0, p, None) == -1


def test_python_front_end_accepts_additive_and_refuses_a_bogus_attention():
    from distributed_sddmm_b200 import driver as D
    assert "additive" in D.GAT.ATTENTIONS
    with pytest.raises(ValueError, match="additive"):
        D.GAT(None, [(4, 4, 1)], attention="Additive")
