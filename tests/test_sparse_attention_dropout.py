"""Attention dropout in fused sparse attention, CPU side: the fp64 model the GPU tests compare against (gradcheck, equal
to the model without dropout at p = 0, the keep statistics of the mask), and the argument validation of the new C entry
points, driver entries and Python front end (no GPU needed)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

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


def test_mix64_is_splitmix64():
    """The restated hash is the splitmix64 generator's output function: seeded with 0, the generator's state after
    k steps is k * 0x9E3779B97F4A7C15 and its first outputs are the published ones."""
    golden = 0x9E3779B97F4A7C15
    states = np.array([(k * golden) % 2 ** 64 for k in range(3)], np.uint64)
    assert [int(x) for x in sd.mix64(states)] == [0xE220A8397B1DCDAF, 0x6E789E6AA1B965F4, 0x06C45D188009454F]


def test_threshold_and_extremes():
    assert sd.threshold(0.0) == 0 and sd.threshold(0.5) == 2 ** 31 and sd.threshold(1 - 2 ** -40) == 2 ** 32 - 1
    assert sd.threshold(0.1) == math.ceil(0.1 * 2 ** 32)
    u, v = np.arange(1000), np.arange(1000)[::-1]
    assert sd.keep(7, 0, u, v, 0.0).all()
    assert not sd.keep(7, 0, u, v, 1 - 2 ** -40).any()


@pytest.mark.parametrize("p", [0.2, 0.6])
def test_model_passes_gradcheck(p):
    rng = np.random.default_rng(5)
    M, N, heads, d = 9, 7, 2, 3
    rows, cols = _pattern(rng, M, N)
    ri, ci = torch.from_numpy(rows), torch.from_numpy(cols)
    assert not sd.keep(3, 0, rows, cols, p).all() and sd.keep(3, 0, rows, cols, p).any()
    args = [torch.tensor(rng.standard_normal((n, heads * d)), requires_grad=True) for n in (M, N, N)]

    def f(Q, K, V):
        return sd.attention_torch(ri, ci, M, Q, K, V, heads, 0.7, p, 3)[0]

    assert torch.autograd.gradcheck(f, args, eps=1e-6, atol=1e-8, rtol=1e-6)


def test_model_at_zero_dropout_is_the_model_without_dropout():
    rng = np.random.default_rng(17)
    M, N, heads, d = 40, 29, 2, 4
    rows, cols = _pattern(rng, M, N)
    Q, K, V, dZ = rng.standard_normal((M, heads * d)), rng.standard_normal((N, heads * d)), \
        rng.standard_normal((N, heads * d)), rng.standard_normal((M, heads * d))
    Z0, L0 = sa.forward_np(rows, cols, M, Q, K, V, heads, 0.5)
    Z, L = sd.forward_np(rows, cols, M, Q, K, V, heads, 0.5, 0.0, 123)
    assert np.array_equal(L, L0) and np.allclose(Z, Z0, rtol=1e-15, atol=1e-15)
    for g, g0 in zip(sd.backward_np(rows, cols, M, Q, K, V, dZ, heads, 0.5, 0.0, 123),
                     sa.backward_np(rows, cols, M, Q, K, V, dZ, heads, 0.5)):
        assert np.allclose(g, g0, rtol=1e-14, atol=1e-14)


def test_model_drops_whole_rows_and_keeps_L():
    """A row whose entries are all dropped gets Z = 0 and the L of all its scores; dropout leaves L alone."""
    rng = np.random.default_rng(2)
    M, N, d = 30, 20, 4
    rows, cols = _pattern(rng, M, N)
    Q, K, V = rng.standard_normal((M, d)), rng.standard_normal((N, d)), rng.standard_normal((N, d))
    p, seed = 0.6, 9
    kept = sd.keep(seed, 0, rows, cols, p)
    dead = [u for u in np.unique(rows) if not kept[rows == u].any()]
    assert dead
    Z, L = sd.forward_np(rows, cols, M, Q, K, V, 1, 0.5, p, seed)
    _, L0 = sa.forward_np(rows, cols, M, Q, K, V, 1, 0.5)
    assert np.array_equal(L, L0) and np.isfinite(L[dead]).all() and not Z[dead].any()


@pytest.mark.parametrize("p", [0.1, 0.6])
def test_keep_fraction(p):
    """Over 2^20 (u, v) pairs the kept fraction is within 5 sigma of 1 - p, and the fraction kept in both of two heads
    within 5 sigma of (1 - p)^2 (the heads' masks are independent)."""
    n = 1 << 20
    rng = np.random.default_rng(1)
    u = rng.integers(0, 1 << 32, n, dtype=np.uint64)
    v = rng.integers(0, 1 << 32, n, dtype=np.uint64)
    # and a dense corner, where u and v differ in their low bits only
    u[: 1 << 16], v[: 1 << 16] = np.repeat(np.arange(256), 256), np.tile(np.arange(256), 256)
    k0, k1 = sd.keep(77, 0, u, v, p), sd.keep(77, 1, u, v, p)
    for frac, q in ((k0.mean(), 1 - p), (k1.mean(), 1 - p), ((k0 & k1).mean(), (1 - p) ** 2)):
        assert abs(frac - q) < 5 * math.sqrt(q * (1 - q) / n), (frac, q)
    # another seed gives another mask
    assert (sd.keep(78, 0, u, v, p) != k0).mean() > 0.1


def test_kernel_entry_points_validate_without_a_gpu(hnh):
    """p < 0, p >= 1, NaN and negative offsets are refused before the device is touched, as are the arguments the
    calls without dropout refuse; empty input is a no-op; a real call fails cleanly without a device."""
    buf = (C.c_double * 8)()
    p = C.addressof(buf)

    def step(rs=p, ci=p, rows=4, nnz=4, d=4, Q=p, ldq=4, K=p, ldk=4, V=p, ldv=4, scale=0.5, acc=p, ldacc=4, m=p, ldm=1,
             s=p, lds=1, pr=0.5, seed=1, u0=0, v0=0):
        return hnh.hnh_sparse_attention_step_dropout_f64(rs, ci, rows, nnz, d, Q, ldq, K, ldk, V, ldv, scale, acc, ldacc, m,
                                                         ldm, s, lds, pr, seed, u0, v0, None)

    def grad_q(rs=p, ci=p, rows=4, nnz=4, d=4, Q=p, ldq=4, dZ=p, lddz=4, L=p, ldl=1, t=p, ldt=1, K=p, ldk=4, V=p, ldv=4,
               scale=0.5, dQ=p, lddq=4, pr=0.5, seed=1, u0=0, v0=0):
        return hnh.hnh_sparse_attention_grad_q_dropout_f64(rs, ci, rows, nnz, d, Q, ldq, dZ, lddz, L, ldl, t, ldt, K, ldk, V,
                                                           ldv, scale, dQ, lddq, pr, seed, u0, v0, None)

    def grad_kv(rs=p, ci=p, rows=4, nnz=4, d=4, K=p, ldk=4, V=p, ldv=4, Q=p, ldq=4, dZ=p, lddz=4, L=p, ldl=1, t=p, ldt=1,
                scale=0.5, dK=p, lddk=4, dV=p, lddv=4, pr=0.5, seed=1, u0=0, v0=0):
        return hnh.hnh_sparse_attention_grad_kv_dropout_f64(rs, ci, rows, nnz, d, K, ldk, V, ldv, Q, ldq, dZ, lddz, L, ldl, t,
                                                            ldt, scale, dK, lddk, dV, lddv, pr, seed, u0, v0, None)

    for call in (step, grad_q, grad_kv):
        for bad in (-0.1, 1.0, 1.5, math.nan, math.inf, -math.inf):
            assert call(pr=bad) == -1
            assert b"dropout probability" in hnh.hnh_last_error_string()
            # refused even where there is nothing to do
            assert call(pr=bad, rows=0) == -1
        assert call(u0=-1) == -1 and call(v0=-1) == -1
        assert b"negative row or column offset" in hnh.hnh_last_error_string()
        assert call(rows=-1) == -1 and call(nnz=-1) == -1 and call(d=0) == -1
        assert call(ldq=3) == -1 and call(ldk=3) == -1 and call(ldv=3) == -1
        for bad in (math.inf, math.nan):
            assert call(scale=bad) == -1
            assert b"scale must be finite" in hnh.hnh_last_error_string()
        assert call(rs=None) == -1 and call(ci=None) == -1 and call(Q=None) == -1 and call(K=None) == -1
        assert call(rs=None, ci=None, Q=None, K=None, V=None, rows=0) == 0
        assert call(rs=None, ci=None, Q=None, K=None, V=None, nnz=0, pr=0.0, seed=2 ** 64 - 1) == 0
    assert step(acc=None) == -1 and step(ldm=0) == -1
    assert grad_q(dQ=None) == -1 and grad_q(ldt=0) == -1
    assert grad_kv(dV=None) == -1 and grad_kv(lddk=3) == -1
    if not torch.cuda.is_available():
        # arguments that pass: the launch needs the device (HNH_E_CUDA), and there is no CPU fallback
        for call in (step, grad_q, grad_kv):
            assert call() == -2
            assert call(pr=0.0) == -2
    # driver entries: null handles and arguments, a non-finite scale
    assert hnh.hnhd_alg_sparse_attention_dropout(None, p, p, p, p, p, 1, 0.5, 0.1, 0) == -1
    assert b"null argument" in hnh.hnh_last_error_string()
    assert hnh.hnhd_alg_sparse_attention_backward_dropout(None, p, p, p, p, p, p, p, p, p, 1, 0.5, 0.1, 0) == -1
    assert b"null argument" in hnh.hnh_last_error_string()


def test_python_front_end_validates_dropout_and_seed():
    from distributed_sddmm_b200 import driver as D
    assert D.Algorithm._dropout_args(0, 0) == (0.0, 0)
    assert D.Algorithm._dropout_args(0.6, 2 ** 64 - 1) == (0.6, 2 ** 64 - 1)
    assert D.Algorithm._dropout_args(0.1, np.uint64(5)) == (0.1, 5)
    for bad in (-0.1, 1.0, math.nan, math.inf):
        with pytest.raises(ValueError, match="must lie in"):
            D.Algorithm._dropout_args(bad, 0)
    for bad in (-1, 2 ** 64, 1.5, "3", True):
        with pytest.raises(ValueError, match="seed"):
            D.Algorithm._dropout_args(0.1, bad)
