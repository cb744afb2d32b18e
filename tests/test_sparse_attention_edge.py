"""Edge features in fused sparse attention, CPU side: the fp64 model the GPU tests compare against (gradcheck in Q, K, V,
E and the bias, equal to the bias model at E = 0 with dE = scale dbias Q_u + D w alpha dZ_u there, equal to dense
masked softmax with keys and values indexed per (u, v)), and the argument validation of the new C entry points, driver
entries and Python front end (no GPU needed)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from tests import sparse_attention_bias_oracle as sb
from tests import sparse_attention_dropout_oracle as sd
from tests import sparse_attention_edge_oracle as se
from tests.test_sparse_attention_bias import _pattern


@pytest.mark.parametrize("p", [0.0, 0.4])
@pytest.mark.parametrize("with_bias", [False, True])
def test_model_passes_gradcheck(p, with_bias):
    rng = np.random.default_rng(7)
    M, N, heads, d = 9, 7, 2, 3
    rows, cols = _pattern(rng, M, N)
    nnz = len(rows)
    ri, ci = torch.from_numpy(rows), torch.from_numpy(cols)
    args = [torch.tensor(rng.standard_normal((n, heads * d)), requires_grad=True) for n in (M, N, N, nnz)]
    args.append(torch.tensor(rng.standard_normal(heads * nnz), requires_grad=with_bias))

    def f(Q, K, V, E, b):
        B = b.reshape(heads, nnz).T if with_bias else torch.zeros(nnz, heads, dtype=torch.float64)
        return se.attention_torch(ri, ci, M, Q, K, V, E, B, heads, 0.7, p, 3)[0]

    assert torch.autograd.gradcheck(f, args, eps=1e-6, atol=1e-8, rtol=1e-6)


def test_model_at_edge_zero_is_the_bias_model():
    """E = 0: Z, L, dQ, dK, dV and dbias of the bias model, and dE = scale dbias Q_u + D w alpha dZ_u."""
    rng = np.random.default_rng(19)
    M, N, heads, d = 40, 29, 2, 4
    r = heads * d
    rows, cols = _pattern(rng, M, N)
    nnz = len(rows)
    Q, K, V, dZ = rng.standard_normal((M, r)), rng.standard_normal((N, r)), rng.standard_normal((N, r)), \
        rng.standard_normal((M, r))
    bias = rng.uniform(-1, 1, heads * nnz)
    bias[rng.random(heads * nnz) < 0.1] = -np.inf
    E0 = np.zeros((nnz, r))
    scale = 0.5
    for p in (0.0, 0.3):
        Z0, L0 = sb.forward_np(rows, cols, M, Q, K, V, bias, heads, scale, p, 123)
        Z, L = se.forward_np(rows, cols, M, Q, K, V, E0, heads, scale, p, 123, bias=bias)
        assert np.array_equal(L, L0) and np.allclose(Z, Z0, rtol=1e-15, atol=1e-15)
        dQ, dK, dV, dE, db = se.backward_np(rows, cols, M, Q, K, V, E0, dZ, heads, scale, p, 123, bias=bias)
        for g, g0 in zip((dQ, dK, dV, db), sb.backward_np(rows, cols, M, Q, K, V, dZ, bias, heads, scale, p, 123)):
            assert np.allclose(g, g0, rtol=1e-14, atol=1e-14)
        w = sd.weights(rows, cols, heads, p, 123) if p > 0 else np.ones((nnz, heads))
        B = sb.bias_matrix(bias, nnz, heads)
        for h in range(heads):
            win = slice(h * d, (h + 1) * d)
            x = scale * (Q[rows, win] * K[cols, win]).sum(1) + B[:, h]
            with np.errstate(invalid="ignore"):  # masked rows: -inf - -inf
                alpha = np.where(np.isneginf(B[:, h]), 0.0, np.exp(x - L[rows, h]))
            want = scale * db.reshape(heads, nnz)[h][:, None] * Q[rows, win] + (w[:, h] * alpha)[:, None] * dZ[rows, win]
            assert np.allclose(dE[:, win], want, rtol=1e-13, atol=1e-13)
            assert not dE[np.isneginf(B[:, h]), win].any()


@pytest.mark.parametrize("heads", [1, 3])
def test_model_matches_dense_masked_softmax_with_per_pair_keys_and_values(heads):
    """Without duplicates, Z_u,h = sum_v softmax_v(scale <Q_u, Kf[u, v]> + B[u, v]) Vf[u, v] with Kf[u, v] = K_v + E_uv and
    Vf[u, v] = V_v + E_uv dense M x N x d tensors, B = -inf off S and on masked entries; the same for L."""
    rng = np.random.default_rng(31 + heads)
    M, N, d = 23, 17, 4
    r = heads * d
    pairs = rng.choice(M * N, 120, replace=False)
    rows, cols = pairs // N, pairs % N
    order = np.lexsort((cols, rows))
    rows, cols = rows[order].astype(np.int64), cols[order].astype(np.int64)
    nnz = len(rows)
    bias = rng.uniform(-3, 3, heads * nnz)
    bias[rng.random(heads * nnz) < 0.15] = -np.inf
    Q, K, V, E = rng.standard_normal((M, r)), rng.standard_normal((N, r)), rng.standard_normal((N, r)), \
        rng.standard_normal((nnz, r))
    scale = 0.6
    Z, L = se.forward_np(rows, cols, M, Q, K, V, E, heads, scale, bias=bias)
    Bm = sb.bias_matrix(bias, nnz, heads)
    for h in range(heads):
        w = slice(h * d, (h + 1) * d)
        B = np.full((M, N), -np.inf)
        B[rows, cols] = Bm[:, h]
        Ef = np.zeros((M, N, d))
        Ef[rows, cols] = E[:, w]
        Kf, Vf = K[None, :, w] + Ef, V[None, :, w] + Ef
        x = scale * np.einsum("uk,uvk->uv", Q[:, w], Kf) + B
        live = np.isfinite(B).any(1)
        xl = torch.from_numpy(x[live])
        a = torch.softmax(xl, 1).numpy()
        want = np.einsum("uv,uvk->uk", a, Vf[live])
        assert np.allclose(Z[live, w], want, rtol=1e-13, atol=1e-13)
        assert np.allclose(L[live, h], torch.logsumexp(xl, 1).numpy(), rtol=1e-13, atol=1e-13)
        assert not Z[~live, w].any() and np.isneginf(L[~live, h]).all()


def test_kernel_entry_points_validate_without_a_gpu(hnh):
    """A null E, lde or ldde below d, dE that is E, a dbias without a bias, p outside [0, 1) and negative offsets are
    refused before the device is touched, as are the arguments the calls without E refuse; a null bias and a null dE
    are accepted; a real call fails cleanly without a device."""
    buf = (C.c_double * 8)()
    p = C.addressof(buf)
    ebuf = (C.c_double * 8)()
    e = C.addressof(ebuf)

    def step(rs=p, ci=p, rows=4, nnz=4, d=4, Q=p, ldq=4, K=p, ldk=4, V=p, ldv=4, scale=0.5, acc=p, ldacc=4, m=p, ldm=1,
             s=p, lds=1, pr=0.5, seed=1, u0=0, v0=0, b=p, db=None, E=e, lde=4, dE=None, ldde=4):
        assert db is None and dE is None
        return hnh.hnh_sparse_attention_step_edge_f64(rs, ci, rows, nnz, d, Q, ldq, K, ldk, V, ldv, scale, acc, ldacc, m, ldm,
                                                      s, lds, pr, seed, u0, v0, b, E, lde, None)

    def grad_q(rs=p, ci=p, rows=4, nnz=4, d=4, Q=p, ldq=4, dZ=p, lddz=4, L=p, ldl=1, t=p, ldt=1, K=p, ldk=4, V=p, ldv=4,
               scale=0.5, dQ=p, lddq=4, pr=0.5, seed=1, u0=0, v0=0, b=p, db=p, E=e, lde=4, dE=p, ldde=4):
        return hnh.hnh_sparse_attention_grad_q_edge_f64(rs, ci, rows, nnz, d, Q, ldq, dZ, lddz, L, ldl, t, ldt, K, ldk, V, ldv,
                                                        scale, dQ, lddq, pr, seed, u0, v0, b, db, E, lde, dE, ldde, None)

    def grad_kv(rs=p, ci=p, rows=4, nnz=4, d=4, K=p, ldk=4, V=p, ldv=4, Q=p, ldq=4, dZ=p, lddz=4, L=p, ldl=1, t=p, ldt=1,
                scale=0.5, dK=p, lddk=4, dV=p, lddv=4, pr=0.5, seed=1, u0=0, v0=0, b=p, db=p, E=e, lde=4, dE=None, ldde=4):
        assert dE is None
        return hnh.hnh_sparse_attention_grad_kv_edge_f64(rs, ci, rows, nnz, d, K, ldk, V, ldv, Q, ldq, dZ, lddz, L, ldl, t,
                                                         ldt, scale, dK, lddk, dV, lddv, pr, seed, u0, v0, b, db, E, lde, None)

    for call in (step, grad_q, grad_kv):
        assert call(E=None) == -1 and b"null E" in hnh.hnh_last_error_string()
        assert call(E=None, rows=0) == -1 and call(E=None, pr=0.0, b=None) == -1
        assert call(lde=3) == -1 and b"lde 3 below d = 4" in hnh.hnh_last_error_string()
        for bad in (-0.1, 1.0, math.nan, math.inf):
            assert call(pr=bad) == -1
            assert b"dropout probability" in hnh.hnh_last_error_string()
        assert call(u0=-1) == -1 and call(v0=-1) == -1
        assert b"negative row or column offset" in hnh.hnh_last_error_string()
        assert call(rows=-1) == -1 and call(nnz=-1) == -1 and call(d=0) == -1
        assert call(ldq=3) == -1 and call(ldk=3) == -1 and call(ldv=3) == -1
        assert call(scale=math.nan) == -1
        assert call(rs=None) == -1 and call(ci=None) == -1 and call(Q=None) == -1
        # a null bias is the call without bias; empty blocks are successful no-ops
        assert call(rs=None, ci=None, Q=None, K=None, V=None, rows=0, b=None, db=None) == 0
        assert call(rs=None, ci=None, Q=None, K=None, V=None, nnz=0, pr=0.0) == 0
    for call in (grad_q, grad_kv):
        assert call(b=None) == -1 and b"dbias without a bias" in hnh.hnh_last_error_string()
    assert grad_q(ldde=3) == -1 and b"ldde 3 below d = 4" in hnh.hnh_last_error_string()
    assert grad_q(dE=e) == -1 and b"dE is E" in hnh.hnh_last_error_string()
    assert grad_q(dE=None, ldde=0, rows=0) == 0
    if not torch.cuda.is_available():
        for call in (step, grad_q, grad_kv):
            assert call() == -2 and call(pr=0.0) == -2 and call(b=None, db=None) == -2
        assert grad_q(dE=None, ldde=0) == -2
    # driver entries: null handles and arguments
    assert hnh.hnhd_alg_sparse_attention_edge(None, p, p, p, p, p, 1, 0.5, 0.0, 0, None, p) == -1
    assert b"null argument" in hnh.hnh_last_error_string()
    assert hnh.hnhd_alg_sparse_attention_edge(p, p, p, None, p, p, 1, 0.5, 0.0, 0, None, p) == -1
    assert hnh.hnhd_alg_sparse_attention_backward_edge(None, p, p, p, p, p, p, p, p, p, 1, 0.5, 0.0, 0, None, None, None,
                                                       None, p, p, None) == -1
    assert b"null argument" in hnh.hnh_last_error_string()
    assert hnh.hnhd_alg_sparse_attention_backward_edge(p, p, p, p, p, p, None, p, p, p, 1, 0.5, 0.0, 0, None, None, None,
                                                       None, p, p, None) == -1


def test_python_front_end_validates_edge_arguments():
    """The front end refuses these arguments before it touches the algorithm's handle (here a null one)."""
    from distributed_sddmm_b200 import driver as D
    alg = D.Algorithm.__new__(D.Algorithm)
    alg.h = None
    bw = D.Algorithm.sparse_attention_backward
    x = object()
    with pytest.raises(ValueError, match="both value orders"):
        bw(alg, x, x, x, x, x, x, x, x, x, 1, 0.5, edge=x)
    with pytest.raises(ValueError, match="both value orders"):
        bw(alg, x, x, x, x, x, x, x, x, x, 1, 0.5, edge_B=x)
    with pytest.raises(ValueError, match="dedge needs the edge features"):
        bw(alg, x, x, x, x, x, x, x, x, x, 1, 0.5, dedge=x)
    with pytest.raises(ValueError, match="both value orders"):
        bw(alg, x, x, x, x, x, x, x, x, x, 1, 0.5, edge=x, edge_B=x, bias=x)
    with pytest.raises(ValueError, match="need their bias"):
        bw(alg, x, x, x, x, x, x, x, x, x, 1, 0.5, edge=x, edge_B=x, dbias=x)
    with pytest.raises(TypeError, match="must be a Dense"):
        D.Algorithm._dense_arg(np.zeros((3, 3)), "edge")
    assert D.Algorithm._dense_arg(None, "edge") is None

