"""Fused sparse attention, CPU side: the fp64 model the GPU tests compare against (checked with gradcheck and against a
dense masked torch.softmax), and the argument validation of the new C entry points and the Python front end (no GPU
needed)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from tests import sparse_attention_oracle as sa


def _pattern(rng, M, N, per_row=4):
    """Rows with empty rows, a duplicate pair and M != N."""
    rows = np.repeat(np.arange(M), rng.integers(0, per_row + 1, M))
    rows = rows[rows % 5 != 3]  # rows 3, 8, ... stay empty
    cols = rng.integers(0, N, len(rows))
    rows = np.concatenate([rows, [0, 0]])
    cols = np.concatenate([cols, [1, 1]])
    return rows.astype(np.int64), cols.astype(np.int64)


def test_model_passes_gradcheck():
    rng = np.random.default_rng(5)
    M, N, heads, d = 9, 7, 2, 3
    rows, cols = _pattern(rng, M, N)
    ri, ci = torch.from_numpy(rows), torch.from_numpy(cols)
    args = [torch.tensor(rng.standard_normal((n, heads * d)), requires_grad=True) for n in (M, N, N)]

    def f(Q, K, V):
        return sa.attention_torch(ri, ci, M, Q, K, V, heads, 0.7)[0]

    assert torch.autograd.gradcheck(f, args, eps=1e-6, atol=1e-8, rtol=1e-6)


@pytest.mark.parametrize("heads", [1, 2, 4])
def test_model_equals_dense_masked_softmax(heads):
    """Z equals torch.softmax(...) @ V over the masked dense scores on rows with entries; rows without entries give
    Z = 0 and L = -inf; L is the rows' log-sum-exp."""
    rng = np.random.default_rng(11 + heads)
    M, N, d = 40, 29, 4
    rows, cols = _pattern(rng, M, N)
    Q, K, V = (rng.standard_normal((n, heads * d)) for n in (M, N, N))
    scale = 1 / math.sqrt(d)
    Z, L = sa.forward_np(rows, cols, M, Q, K, V, heads, scale)
    want = sa.dense_masked_np(rows, cols, M, N, Q, K, V, heads, scale)
    assert np.abs(want).max() > 0
    assert np.allclose(Z, want, rtol=1e-12, atol=1e-14)
    empty = np.setdiff1d(np.arange(M), rows)
    assert len(empty) and not Z[empty].any() and np.isneginf(L[empty]).all()
    for h in range(heads):
        w = slice(h * d, (h + 1) * d)
        x = scale * (Q[rows, w] * K[cols, w]).sum(1)
        lse = np.full(M, -np.inf)
        for u in np.unique(rows):
            lse[u] = np.log(np.exp(x[rows == u]).sum())
        assert np.allclose(L[:, h], lse, rtol=1e-13, atol=0)


def test_model_is_finite_for_large_scores():
    rng = np.random.default_rng(3)
    M, N = 6, 5
    rows, cols = _pattern(rng, M, N)
    Q = rng.choice([-1.0, 1.0], (M, 4)) * 1000
    K = rng.choice([-1.0, 1.0], (N, 4))
    V = rng.standard_normal((N, 4))
    Z, _ = sa.forward_np(rows, cols, M, Q, K, V, 1, 0.25)
    assert np.isfinite(Z).all()
    dQ, dK, dV = sa.backward_np(rows, cols, M, Q, K, V, np.ones((M, 4)), 1, 0.25)
    assert np.isfinite(dQ).all() and np.isfinite(dK).all() and np.isfinite(dV).all()


def test_kernel_entry_points_validate_without_a_gpu(hnh):
    """Null pointers, negative sizes, d < 1, leading dimensions below d (rows) or 1 (scalars) and a non-finite scale
    are refused before the device is touched; empty input is a no-op."""
    buf = (C.c_double * 8)()
    p = C.addressof(buf)

    def step(rs=p, ci=p, rows=4, nnz=4, d=4, Q=p, ldq=4, K=p, ldk=4, V=p, ldv=4, scale=0.5, acc=p, ldacc=4, m=p, ldm=1,
             s=p, lds=1):
        return hnh.hnh_sparse_attention_step_f64(rs, ci, rows, nnz, d, Q, ldq, K, ldk, V, ldv, scale, acc, ldacc, m, ldm, s,
                                                 lds, None)

    def grad_q(rs=p, ci=p, rows=4, nnz=4, d=4, Q=p, ldq=4, dZ=p, lddz=4, L=p, ldl=1, t=p, ldt=1, K=p, ldk=4, V=p, ldv=4,
               scale=0.5, dQ=p, lddq=4):
        return hnh.hnh_sparse_attention_grad_q_f64(rs, ci, rows, nnz, d, Q, ldq, dZ, lddz, L, ldl, t, ldt, K, ldk, V, ldv,
                                                   scale, dQ, lddq, None)

    def grad_kv(rs=p, ci=p, rows=4, nnz=4, d=4, K=p, ldk=4, V=p, ldv=4, Q=p, ldq=4, dZ=p, lddz=4, L=p, ldl=1, t=p, ldt=1,
                scale=0.5, dK=p, lddk=4, dV=p, lddv=4):
        return hnh.hnh_sparse_attention_grad_kv_f64(rs, ci, rows, nnz, d, K, ldk, V, ldv, Q, ldq, dZ, lddz, L, ldl, t, ldt,
                                                    scale, dK, lddk, dV, lddv, None)

    for call in (step, grad_q, grad_kv):
        assert call(rows=-1) == -1
        assert call(nnz=-1) == -1
        assert call(d=0) == -1
        assert b"d must be positive" in hnh.hnh_last_error_string()
        assert call(ldq=3) == -1
        assert b"leading dimension" in hnh.hnh_last_error_string()
        assert call(ldk=3) == -1
        assert call(ldv=3) == -1
        for bad in (math.inf, -math.inf, math.nan):
            assert call(scale=bad) == -1
            assert b"scale must be finite" in hnh.hnh_last_error_string()
        assert call(rs=None) == -1
        assert b"null pointer" in hnh.hnh_last_error_string()
        assert call(ci=None) == -1
        assert call(Q=None) == -1
        assert call(K=None) == -1
        assert call(V=None) == -1
        # empty blocks: nothing to do, nothing touched
        assert call(rs=None, ci=None, Q=None, K=None, V=None, rows=0) == 0
        assert call(rs=None, ci=None, Q=None, K=None, V=None, nnz=0) == 0
    assert step(acc=None) == -1 and step(m=None) == -1 and step(s=None) == -1
    assert step(ldacc=3) == -1 and step(ldm=0) == -1 and step(lds=0) == -1
    assert grad_q(dZ=None) == -1 and grad_q(L=None) == -1 and grad_q(t=None) == -1 and grad_q(dQ=None) == -1
    assert grad_q(lddz=3) == -1 and grad_q(ldl=0) == -1 and grad_q(ldt=0) == -1 and grad_q(lddq=3) == -1
    assert grad_kv(dZ=None) == -1 and grad_kv(dK=None) == -1 and grad_kv(dV=None) == -1 and grad_kv(L=None) == -1
    assert grad_kv(lddk=3) == -1 and grad_kv(lddv=3) == -1 and grad_kv(ldt=0) == -1

    def finish(rows=4, d=4, acc=p, ldacc=4, m=p, ldm=1, s=p, lds=1, Z=p, ldz=4, L=p, ldl=1):
        return hnh.hnh_sparse_attention_finish_f64(rows, d, acc, ldacc, m, ldm, s, lds, Z, ldz, L, ldl, None)

    assert finish(rows=-1) == -1
    assert finish(d=0) == -1
    assert finish(ldacc=3) == -1 and finish(ldz=3) == -1 and finish(ldm=0) == -1 and finish(lds=0) == -1
    assert finish(ldl=0) == -1
    assert finish(acc=None) == -1 and finish(Z=None) == -1 and finish(L=None) == -1
    assert finish(rows=0, acc=None, m=None, s=None, Z=None, L=None) == 0
    # driver entries: null handles and arguments, a non-finite scale
    assert hnh.hnhd_alg_sparse_attention(None, p, p, p, p, p, 1, 0.5) == -1
    assert b"null argument" in hnh.hnh_last_error_string()
    assert hnh.hnhd_alg_sparse_attention_backward(None, p, p, p, p, p, p, p, p, p, 1, 0.5) == -1
    assert b"null argument" in hnh.hnh_last_error_string()


def test_python_front_end_default_scale_and_heads():
    """scale=None is 1/sqrt(d) with d = r / heads; heads must divide r."""
    from distributed_sddmm_b200 import driver as D

    class Shaped:
        shape = (10, 12)

    assert D.Algorithm._attention_scale(Shaped(), 1, None) == 1 / math.sqrt(12)
    assert D.Algorithm._attention_scale(Shaped(), 4, None) == 1 / math.sqrt(3)
    assert D.Algorithm._attention_scale(Shaped(), 5, 0.25) == 0.25
    for heads in (5, 0):
        with pytest.raises(ValueError, match="must divide"):
            D.Algorithm._attention_scale(Shaped(), heads, None)
