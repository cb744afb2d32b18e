"""Additive score bias in fused sparse attention, CPU side: the fp64 model the GPU tests compare against (gradcheck in
Q, K, V and the bias, equal to the model without bias at bias 0, equal to dense masked softmax and to
scaled_dot_product_attention with a float attn_mask, masked rows), and the argument validation of the new C entry
points, driver entries and Python front end (no GPU needed)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from tests import sparse_attention_bias_oracle as sb
from tests import sparse_attention_dropout_oracle as sd
from tests import sparse_attention_oracle as sa


def _pattern(rng, M, N, per_row=4):
    """Rows with empty rows, a duplicate pair and M != N."""
    rows = np.repeat(np.arange(M), rng.integers(0, per_row + 1, M))
    rows = rows[rows % 5 != 3]
    cols = rng.integers(0, N, len(rows))
    rows = np.concatenate([rows, [0, 0]])
    cols = np.concatenate([cols, [1, 1]])
    return rows.astype(np.int64), cols.astype(np.int64)


@pytest.mark.parametrize("p", [0.0, 0.4])
@pytest.mark.parametrize("shared", [False, True])
def test_model_passes_gradcheck(p, shared):
    rng = np.random.default_rng(5)
    M, N, heads, d = 9, 7, 2, 3
    rows, cols = _pattern(rng, M, N)
    nnz = len(rows)
    ri, ci = torch.from_numpy(rows), torch.from_numpy(cols)
    args = [torch.tensor(rng.standard_normal((n, heads * d)), requires_grad=True) for n in (M, N, N)]
    args.append(torch.tensor(rng.standard_normal(nnz if shared else heads * nnz), requires_grad=True))

    def f(Q, K, V, b):
        B = b[:, None].expand(nnz, heads) if shared else b.reshape(heads, nnz).T
        return sb.attention_torch(ri, ci, M, Q, K, V, B, heads, 0.7, p, 3)[0]

    assert torch.autograd.gradcheck(f, args, eps=1e-6, atol=1e-8, rtol=1e-6)


def test_model_at_bias_zero_is_the_model_without_bias():
    rng = np.random.default_rng(17)
    M, N, heads, d = 40, 29, 2, 4
    rows, cols = _pattern(rng, M, N)
    Q, K, V, dZ = rng.standard_normal((M, heads * d)), rng.standard_normal((N, heads * d)), \
        rng.standard_normal((N, heads * d)), rng.standard_normal((M, heads * d))
    zero = np.zeros(len(rows))
    for p in (0.0, 0.3):
        Z0, L0 = sd.forward_np(rows, cols, M, Q, K, V, heads, 0.5, p, 123)
        Z, L = sb.forward_np(rows, cols, M, Q, K, V, zero, heads, 0.5, p, 123)
        assert np.array_equal(L, L0) and np.allclose(Z, Z0, rtol=1e-15, atol=1e-15)
        got = sb.backward_np(rows, cols, M, Q, K, V, dZ, zero, heads, 0.5, p, 123)
        for g, g0 in zip(got[:3], sd.backward_np(rows, cols, M, Q, K, V, dZ, heads, 0.5, p, 123)):
            assert np.allclose(g, g0, rtol=1e-14, atol=1e-14)


def _dense_bias(rows, cols, M, N, bias_e):
    """The M x N bias of a pattern without duplicates, -inf off the pattern."""
    B = np.full((M, N), -np.inf)
    B[rows, cols] = bias_e
    return B


@pytest.mark.parametrize("heads", [1, 3])
def test_model_matches_dense_masked_softmax_and_sdpa(heads):
    """Without duplicates, Z_u,h = softmax_v(scale Q K^T + B)[u] V, with B = -inf off S and on masked entries; the same
    as torch's scaled_dot_product_attention with a float attn_mask (rows with at least one live entry)."""
    rng = np.random.default_rng(3 + heads)
    M, N, d = 23, 17, 4
    r = heads * d
    pairs = rng.choice(M * N, 120, replace=False)
    rows, cols = pairs // N, pairs % N
    order = np.lexsort((cols, rows))
    rows, cols = rows[order].astype(np.int64), cols[order].astype(np.int64)
    nnz = len(rows)
    bias = rng.uniform(-3, 3, heads * nnz)
    bias[rng.random(heads * nnz) < 0.15] = -np.inf
    Q, K, V = rng.standard_normal((M, r)), rng.standard_normal((N, r)), rng.standard_normal((N, r))
    scale = 0.6
    Z, L = sb.forward_np(rows, cols, M, Q, K, V, bias, heads, scale)
    Bm = sb.bias_matrix(bias, nnz, heads)
    for h in range(heads):
        w = slice(h * d, (h + 1) * d)
        B = torch.from_numpy(_dense_bias(rows, cols, M, N, Bm[:, h]))
        live = torch.isfinite(B).any(1)
        x = scale * sa._t(Q)[:, w] @ sa._t(K)[:, w].T + B
        want = torch.softmax(x[live], 1) @ sa._t(V)[:, w]
        assert np.allclose(Z[live.numpy(), w], want.numpy(), rtol=1e-13, atol=1e-13)
        assert not Z[~live.numpy(), w].any() and np.isneginf(L[~live.numpy(), h]).all()
        assert np.allclose(L[live.numpy(), h], torch.logsumexp(x[live], 1).numpy(), rtol=1e-13, atol=1e-13)
        sdpa = torch.nn.functional.scaled_dot_product_attention(
            sa._t(Q)[None, live, w], sa._t(K)[None, :, w], sa._t(V)[None, :, w], attn_mask=B[None, live], scale=scale)[0]
        assert np.allclose(Z[live.numpy(), w], sdpa.numpy(), rtol=1e-12, atol=1e-12)


def test_model_masked_rows_have_zero_output_and_finite_gradients():
    """Rows masked throughout: Z = 0, L = -inf, and every gradient (dQ, dK, dV, dbias) finite; a masked entry's dbias
    is 0; large biases (+-800) stay exact through the max shift."""
    rng = np.random.default_rng(11)
    M, N, heads, d = 30, 20, 2, 4
    rows, cols = _pattern(rng, M, N)
    nnz = len(rows)
    Q, K, V, dZ = rng.standard_normal((M, 8)), rng.standard_normal((N, 8)), rng.standard_normal((N, 8)), \
        rng.standard_normal((M, 8))
    bias = rng.uniform(-1, 1, heads * nnz)
    dead = np.unique(rows)[::3]
    Bm = bias.reshape(heads, nnz)
    Bm[:, np.isin(rows, dead)] = -np.inf
    Bm[0, rows % 7 == 1] += 800.0
    Bm[1, rows % 7 == 2] -= 800.0
    bias = Bm.reshape(-1)
    Z, L = sb.forward_np(rows, cols, M, Q, K, V, bias, heads, 0.5, 0.2, 4)
    assert not Z[dead].any() and np.isneginf(L[dead]).all()
    grads = sb.backward_np(rows, cols, M, Q, K, V, dZ, bias, heads, 0.5, 0.2, 4)
    assert all(np.isfinite(g).all() for g in grads)
    assert not grads[3][np.isneginf(bias)].any()
    # the +-800 shift: a bias constant over a row does not change Z
    shift = np.where(np.isfinite(Bm), Bm + np.where(rows % 2 == 0, 800.0, -800.0)[None, :], -np.inf).reshape(-1)
    Z2, L2 = sb.forward_np(rows, cols, M, Q, K, V, shift, heads, 0.5, 0.2, 4)
    assert np.allclose(Z2, Z, rtol=1e-12, atol=1e-12)


def test_kernel_entry_points_validate_without_a_gpu(hnh):
    """A null bias, p outside [0, 1), NaN and negative offsets are refused before the device is touched, as are the
    arguments the calls without bias refuse; a real call fails cleanly without a device."""
    buf = (C.c_double * 8)()
    p = C.addressof(buf)

    def step(rs=p, ci=p, rows=4, nnz=4, d=4, Q=p, ldq=4, K=p, ldk=4, V=p, ldv=4, scale=0.5, acc=p, ldacc=4, m=p, ldm=1,
             s=p, lds=1, pr=0.5, seed=1, u0=0, v0=0, b=p):
        return hnh.hnh_sparse_attention_step_bias_f64(rs, ci, rows, nnz, d, Q, ldq, K, ldk, V, ldv, scale, acc, ldacc, m, ldm,
                                                      s, lds, pr, seed, u0, v0, b, None)

    def grad_q(rs=p, ci=p, rows=4, nnz=4, d=4, Q=p, ldq=4, dZ=p, lddz=4, L=p, ldl=1, t=p, ldt=1, K=p, ldk=4, V=p, ldv=4,
               scale=0.5, dQ=p, lddq=4, pr=0.5, seed=1, u0=0, v0=0, b=p, db=p):
        return hnh.hnh_sparse_attention_grad_q_bias_f64(rs, ci, rows, nnz, d, Q, ldq, dZ, lddz, L, ldl, t, ldt, K, ldk, V, ldv,
                                                        scale, dQ, lddq, pr, seed, u0, v0, b, db, None)

    def grad_kv(rs=p, ci=p, rows=4, nnz=4, d=4, K=p, ldk=4, V=p, ldv=4, Q=p, ldq=4, dZ=p, lddz=4, L=p, ldl=1, t=p, ldt=1,
                scale=0.5, dK=p, lddk=4, dV=p, lddv=4, pr=0.5, seed=1, u0=0, v0=0, b=p, db=p):
        return hnh.hnh_sparse_attention_grad_kv_bias_f64(rs, ci, rows, nnz, d, K, ldk, V, ldv, Q, ldq, dZ, lddz, L, ldl, t,
                                                         ldt, scale, dK, lddk, dV, lddv, pr, seed, u0, v0, b, db, None)

    for call in (step, grad_q, grad_kv):
        assert call(b=None) == -1
        assert b"null bias" in hnh.hnh_last_error_string()
        assert call(b=None, rows=0) == -1 and call(b=None, pr=0.0) == -1
        for bad in (-0.1, 1.0, math.nan, math.inf):
            assert call(pr=bad) == -1
            assert b"dropout probability" in hnh.hnh_last_error_string()
        assert call(u0=-1) == -1 and call(v0=-1) == -1
        assert b"negative row or column offset" in hnh.hnh_last_error_string()
        assert call(rows=-1) == -1 and call(nnz=-1) == -1 and call(d=0) == -1
        assert call(ldq=3) == -1 and call(ldk=3) == -1 and call(ldv=3) == -1
        assert call(scale=math.nan) == -1
        assert call(rs=None) == -1 and call(ci=None) == -1 and call(Q=None) == -1
        assert call(rs=None, ci=None, Q=None, K=None, V=None, rows=0) == 0
        assert call(rs=None, ci=None, Q=None, K=None, V=None, nnz=0, pr=0.0) == 0
    assert grad_q(db=None, rows=0) == 0 and grad_kv(db=None, nnz=0) == 0
    if not torch.cuda.is_available():
        for call in (step, grad_q, grad_kv):
            assert call() == -2 and call(pr=0.0) == -2
        assert grad_q(db=None) == -2 and grad_kv(db=None) == -2
    assert hnh.hnh_entry_coords_from_index_f64(None, None, -1, 0, None) == -1
    assert hnh.hnh_entry_coords_from_index_f64(None, None, 0, 0, None) == 0
    assert hnh.hnh_entry_coords_from_index_f64(p, None, 4, 0, None) == -1
    # driver entries: null handles and arguments
    assert hnh.hnhd_alg_sparse_attention_bias(None, p, p, p, p, p, 1, 0.5, 0.0, 0, p) == -1
    assert b"null argument" in hnh.hnh_last_error_string()
    assert hnh.hnhd_alg_sparse_attention_backward_bias(None, p, p, p, p, p, p, p, p, p, 1, 0.5, 0.0, 0, p, p, None, None) == -1
    assert b"null argument" in hnh.hnh_last_error_string()
    assert hnh.hnhd_alg_entry_coordinates(None, 0, p, p) == -1
    assert b"null argument" in hnh.hnh_last_error_string()


def test_python_front_end_validates_bias_arguments():
    """The front end refuses these arguments before it touches the algorithm's handle (here a null one)."""
    from distributed_sddmm_b200 import driver as D
    alg = D.Algorithm.__new__(D.Algorithm)
    alg.h = None
    bw = D.Algorithm.sparse_attention_backward
    x = object()
    with pytest.raises(ValueError, match="need their bias"):
        bw(alg, x, x, x, x, x, x, x, x, x, 1, 0.5, dbias=x)
    with pytest.raises(ValueError, match="need their bias"):
        bw(alg, x, x, x, x, x, x, x, x, x, 1, 0.5, dbias_B=x)
    with pytest.raises(ValueError, match="both value orders"):
        bw(alg, x, x, x, x, x, x, x, x, x, 1, 0.5, bias=x)
    with pytest.raises(ValueError, match="both value orders"):
        bw(alg, x, x, x, x, x, x, x, x, x, 1, 0.5, bias_B=x)
    with pytest.raises(TypeError, match="must be a Vec"):
        D.Algorithm._vec_arg(np.zeros(3), "bias")
    assert D.Algorithm._vec_arg(None, "bias") is None
