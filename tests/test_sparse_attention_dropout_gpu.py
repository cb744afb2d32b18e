"""Attention dropout in fused sparse attention on the GPU at p = 1: the three dropout kernels against the fp64 model of
tests/sparse_attention_dropout_oracle.py on every width path, leading dimension, packed form and alignment, with block
offsets past 2^31, past one resident wave, with the online-softmax state carried across two calls and on scores far
below zero; at dropout 0 they are bit-identical to the kernels without dropout.  Algorithm.sparse_attention /
sparse_attention_backward with dropout on every algorithm against the model.  Multi-rank cases live in
tests/test_sparse_attention_dropout_multirank_gpu.py."""
import math

import numpy as np
import pytest

from distributed_sddmm_b200 import driver as D
from tests import sparse_attention_dropout_oracle as sd
from tests.kernel_waves_worker import CTAS_PER_SM
from tests.mp_edge_softmax_worker import coords
from tests.test_sparse_attention_gpu import ALGS, WIDTHS, Side, _algorithm, _block, _csr, _dense, _ptrs, rel_err

pytestmark = pytest.mark.gpu
SEED = 0xC0FFEE + 31
KERNEL_TOL = 1e-12
# global offsets of the test block: past 2^31, so the mask sees S-rows and S-columns with their top bit set
U0, V0 = 3_000_000_000, 2_500_000_123


@pytest.fixture(scope="module")
def world():
    D.world_init("self")
    yield
    D.world_finalize()


def _run(L, st, rs, ci, rsT, ciT, M, N, nnz, d, scale, Qv, Kv, Vv, dZv, dQ0, dK0, dV0, Lw, t_np, layout, drop):
    """Forward (step + finish in place), grad_q on the block and grad_kv on its transpose; drop = (p, seed, u0, v0)
    for the dropout entry points, None for the ones without.  Returns Z, L, dQ - dQ0, dK - dK0, dV - dV0."""
    import torch
    packed, extra, shift = layout
    zeros = lambda n, w: np.zeros((n, w))  # noqa: E731
    tail = () if drop is None else tuple(drop)
    sfx = "_f64" if drop is None else "_dropout_f64"
    fn = lambda name: getattr(L, "hnh_sparse_attention_" + name + sfx)  # noqa: E731
    R = Side(M, [("Q", Qv), ("acc", zeros(M, d)), ("m", np.full((M, 1), np.nan)), ("s", zeros(M, 1))], packed, extra, shift)
    Y = Side(N, [("K", Kv), ("V", Vv)], packed, extra, shift)
    D.check(fn("step")(rs, ci, M, nnz, d, *_ptrs(R, "Q"), *_ptrs(Y, "K", "V"), scale, *_ptrs(R, "acc", "m", "s"), *tail, st))
    D.check(L.hnh_sparse_attention_finish_f64(M, d, *_ptrs(R, "acc", "m", "s"), *_ptrs(R, "acc", "m"), st))
    Rq = Side(M, [("Q", Qv), ("dZ", dZv), ("L", Lw), ("t", t_np), ("dQ", dQ0)], packed, extra, shift)
    D.check(fn("grad_q")(rs, ci, M, nnz, d, *_ptrs(Rq, "Q", "dZ", "L", "t"), *_ptrs(Y, "K", "V"), scale, *_ptrs(Rq, "dQ"),
                         *tail, st))
    Rk = Side(N, [("K", Kv), ("V", Vv), ("dK", dK0), ("dV", dV0)], packed, extra, shift)
    Yq = Side(M, [("Q", Qv), ("dZ", dZv), ("L", Lw), ("t", t_np)], packed, extra, shift)
    D.check(fn("grad_kv")(rsT, ciT, N, nnz, d, *_ptrs(Rk, "K", "V"), *_ptrs(Yq, "Q", "dZ", "L", "t"), scale,
                          *_ptrs(Rk, "dK", "dV"), *tail, st))
    torch.cuda.synchronize()
    return (R.get("acc"), R.get("m")[:, 0], Rq.get("dQ") - dQ0, Rk.get("dK") - dK0, Rk.get("dV") - dV0)


def _check(rowStart, rr, cc, M, N, d, rng, layouts, p, seed=SEED, scale=None, QK=None, u0=U0, v0=V0):
    """The dropout kernels against the model on every layout (packed, extra, shift); at p = 0 also bit-identical to
    the kernels without dropout."""
    import torch
    from distributed_sddmm_b200 import lib
    L = lib()
    st = torch.cuda.current_stream().cuda_stream
    scale = 1 / math.sqrt(d) if scale is None else scale
    Qv, dZv, dQ0 = (rng.uniform(-1, 1, (M, d)) for _ in range(3))
    Kv, Vv, dK0, dV0 = (rng.uniform(-1, 1, (N, d)) for _ in range(4))
    if QK is not None:
        Qv, Kv = QK
    Zw, Lw = sd.forward_np(rr, cc, M, Qv, Kv, Vv, 1, scale, p, seed, u0, v0)
    dQw, dKw, dVw = sd.backward_np(rr, cc, M, Qv, Kv, Vv, dZv, 1, scale, p, seed, u0, v0)
    t_np = (dZv * Zw).sum(1, keepdims=True)
    Lw = Lw.reshape(M, 1)
    dev = lambda x: torch.from_numpy(x).to("cuda:0")  # noqa: E731
    order = np.argsort(cc, kind="stable")
    rsT, _, ciT = _csr(cc[order], rr[order], N)
    ptrs = [dev(x) for x in (rowStart, cc, rsT, ciT)]
    args = [x.data_ptr() for x in ptrs] + [M, N, len(cc), d, scale, Qv, Kv, Vv, dZv, dQ0, dK0, dV0, Lw, t_np]
    want = (Zw, Lw[:, 0], dQw, dKw, dVw)
    for layout in layouts:
        got = _run(L, st, *args, layout, (p, seed, u0, v0))
        for g, w, name in zip(got, want, ("Z", "L", "dQ", "dK", "dV")):
            assert rel_err(g, w) < KERNEL_TOL, (d, layout, p, name)
        if p == 0.0:
            old = _run(L, st, *args, layout, None)
            for g, o, name in zip(got, old, ("Z", "L", "dQ", "dK", "dV")):
                assert np.array_equal(g, o, equal_nan=True), (d, layout, name)
    return Zw


LAYOUTS = ((False, 0, 0), (False, 2, 0), (True, 0, 0), (False, 0, 1))


@pytest.mark.parametrize("d", WIDTHS)
def test_dropout_kernels_match_the_model_on_every_width(world, d):
    """Every width path (4..256 and 7 through the generic kernels) at p = 0.6 and 0.1, on separate operands at
    leading dimension d and d + 2, the packed forms and operands one double off 16-byte alignment (the generic
    kernels); rows of one entry, a row of 1500 entries, duplicate pairs, rows whose entries are all dropped."""
    rng = np.random.default_rng(SEED + d)
    M, N = 301, 257
    rowStart, rr, cc = _block(rng, M, N)
    kept = sd.keep(SEED, 0, rr + U0, cc + V0, 0.6)
    lens = np.diff(rowStart)
    assert any(lens[u] > 0 and not kept[rowStart[u]:rowStart[u + 1]].any() for u in range(M))
    Zw = _check(rowStart, rr, cc, M, N, d, rng, LAYOUTS, 0.6)
    assert np.isfinite(Zw).all()
    _check(rowStart, rr, cc, M, N, d, rng, LAYOUTS[:1], 0.1)


@pytest.mark.parametrize("d", WIDTHS)
def test_dropout_at_zero_is_bit_identical_to_the_kernels_without_dropout(world, d):
    rng = np.random.default_rng(SEED + 50 + d)
    M, N = 301, 257
    rowStart, rr, cc = _block(rng, M, N)
    _check(rowStart, rr, cc, M, N, d, rng, (LAYOUTS[0], LAYOUTS[3]), 0.0)


@pytest.mark.parametrize("d", WIDTHS)
def test_dropout_kernels_on_large_scores(world, d):
    """Rows whose scores all lie near -800 or +800, of every length from 1 to 40 (most chunks part-full), as in
    test_sparse_attention_gpu.py: exact only if every chunk is shifted by the maximum of its own entries, dropped
    entries included."""
    rng = np.random.default_rng(SEED + 300 + d)
    M, N = 164, 64
    lens = np.arange(M) % 41
    rowStart = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    rr = np.repeat(np.arange(M), lens).astype(np.int64)
    cc = rng.integers(0, N, len(rr)).astype(np.int64)
    sign = np.where(np.arange(M) % 2 == 0, -1.0, 1.0)
    Qv = (sign * 100.0)[:, None] * np.ones((1, d))
    w = np.zeros((N, d))
    for i in range(d // 2):
        r = ((np.arange(N) + i) % 7 - 3).astype(np.float64)
        w[:, 2 * i], w[:, 2 * i + 1] = r, -r
    Kv = (8.0 + (np.arange(N) % 8) / 64.0)[:, None] + w
    scale = 2.0 ** -math.floor(math.log2(d))
    assert (np.abs(scale * (Qv[rr] * Kv[cc]).sum(1)) > 745).all()
    _check(rowStart, rr, cc, M, N, d, rng, (LAYOUTS[0], LAYOUTS[2], LAYOUTS[3]), 0.3, scale=scale, QK=(Qv, Kv))


@pytest.mark.parametrize("d", [4, 64, 7])
def test_dropout_kernels_past_one_resident_wave(world, d):
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rows_per_cta = 256 // {4: 2, 64: 32}.get(d, 32)
    M = 3 * CTAS_PER_SM * sms * rows_per_cta + 5
    rng = np.random.default_rng(SEED + 100 + d)
    lens = rng.integers(0, 4, M)
    rowStart = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    rr = np.repeat(np.arange(M), lens)
    cc = rng.integers(0, M, len(rr)).astype(np.int64)
    _check(rowStart, rr, cc, M, M, d, rng, LAYOUTS[:1], 0.5, u0=0, v0=0)


@pytest.mark.parametrize("d", [8, 128, 7])
def test_dropout_state_carries_across_two_calls(world, d):
    """One block fed as two calls (its entries with v < N/2, then the rest, each call with the same offsets) equals
    one call and the model: the mask follows (u, v), not the entries' positions."""
    import torch
    from distributed_sddmm_b200 import lib
    L = lib()
    st = torch.cuda.current_stream().cuda_stream
    rng = np.random.default_rng(SEED + 200 + d)
    M, N = 301, 257
    rowStart, rr, cc = _block(rng, M, N)
    Qv, Kv, Vv = rng.uniform(-1, 1, (M, d)), rng.uniform(-1, 1, (N, d)), rng.uniform(-1, 1, (N, d))
    Y = Side(N, [("K", Kv), ("V", Vv)])
    dev = lambda x: torch.from_numpy(x).to("cuda:0")  # noqa: E731
    scale, p = 1 / math.sqrt(d), 0.4
    drop = (p, SEED, U0, V0)

    def state():
        return Side(M, [("Q", Qv), ("acc", np.zeros((M, d))), ("m", np.full((M, 1), np.nan)), ("s", np.zeros((M, 1)))])

    def run(parts, S):
        for rs, ci, n in parts:
            D.check(L.hnh_sparse_attention_step_dropout_f64(rs.data_ptr(), ci.data_ptr(), M, n, d, *_ptrs(S, "Q"),
                                                            *_ptrs(Y, "K", "V"), scale, *_ptrs(S, "acc", "m", "s"), *drop, st))
        D.check(L.hnh_sparse_attention_finish_f64(M, d, *_ptrs(S, "acc", "m", "s"), *_ptrs(S, "acc", "m"), st))

    one, two = state(), state()
    run([(dev(rowStart), dev(cc), len(cc))], one)
    halves = []
    for keep in (cc < N // 2, cc >= N // 2):
        r2, _, c2 = _csr(rr[keep], cc[keep], M)
        halves.append((dev(r2), dev(c2), int(keep.sum())))
    run(halves, two)
    torch.cuda.synchronize()
    assert rel_err(two.get("acc"), one.get("acc")) < 1e-14
    assert rel_err(two.get("m"), one.get("m")) < 1e-14
    Zw, Lw = sd.forward_np(rr, cc, M, Qv, Kv, Vv, 1, scale, p, SEED, U0, V0)
    assert rel_err(two.get("acc"), Zw) < KERNEL_TOL and rel_err(two.get("m")[:, 0], Lw[:, 0]) < KERNEL_TOL


# ---- Algorithm.sparse_attention / sparse_attention_backward with dropout at p = 1 ---------------------------------------
@pytest.mark.parametrize("shape", ["square", "rectangular"])
@pytest.mark.parametrize("name", ALGS)
def test_p1_algorithm_with_dropout(world, name, shape):
    """Every algorithm, 1 and 2 heads, dropout 0.1 and 0.6: Z, L, dQ, dK and dV against the model within 1e-10; a
    repeat is bit-identical, another seed gives another Z, and dropout 0 equals the call without dropout bit for
    bit."""
    for heads in (1, 2):
        d = 4
        r = heads * d
        S, alg = _algorithm(name, shape, r)
        dims = alg.dims
        Ma, Nb = dims.localArows, dims.localBrows
        rows, cols = coords(alg, "A")
        rng = np.random.default_rng(SEED + heads)
        Qv, dZv = rng.uniform(-1, 1, (Ma, r)), rng.uniform(-1, 1, (Ma, r))
        Kv, Vv = rng.uniform(-1, 1, (Nb, r)), rng.uniform(-1, 1, (Nb, r))
        Q, K, V, dZ = _dense(alg, "A", Qv), _dense(alg, "B", Kv), _dense(alg, "B", Vv), _dense(alg, "A", dZv)
        Z, Lm = alg.like_A_matrix(np.nan), D.Dense.create(Ma, heads, np.nan)
        dQ, dK, dV = alg.like_A_matrix(np.nan), alg.like_B_matrix(np.nan), alg.like_B_matrix(np.nan)
        scale = 1 / math.sqrt(d)

        def run(**kw):
            alg.sparse_attention(Q, K, V, Z, Lm, heads, **kw)
            alg.sparse_attention_backward(Q, K, V, Z, Lm, dZ, dQ, dK, dV, heads, **kw)
            return tuple(m.to_host() for m in (Z, Lm, dQ, dK, dV))

        for p in (0.1, 0.6):
            seed = 1000 + heads
            Zw, Lw = sd.forward_np(rows, cols, Ma, Qv, Kv, Vv, heads, scale, p, seed)
            grads = sd.backward_np(rows, cols, Ma, Qv, Kv, Vv, dZv, heads, scale, p, seed)
            got = run(dropout=p, seed=seed)
            where = (name, shape, heads, p)
            for g, w in zip(got, (Zw, Lw, *grads)):
                assert rel_err(g, w) < 1e-10, where
            assert all(np.array_equal(a, b) for a, b in zip(got, run(dropout=p, seed=seed))), where
            assert not np.array_equal(got[0], run(dropout=p, seed=seed + 7)[0]), where
        base = run()
        assert all(np.array_equal(a, b) for a, b in zip(base, run(dropout=0.0, seed=5))), (name, shape, heads)
        del S, alg


def test_p1_dropout_validation(world):
    """Bad dropout probabilities are refused by the driver entries (HNH_E_INVALID) and the Python front end."""
    from distributed_sddmm_b200 import lib
    d = 8
    S, alg = _algorithm("15d_fusion2", "square", d)
    dims = alg.dims
    Q, K, V = alg.like_A_matrix(0.5), alg.like_B_matrix(0.5), alg.like_B_matrix(0.5)
    Z, Lm = alg.like_A_matrix(), D.Dense.create(dims.localArows, 1)
    dQ, dK, dV = alg.like_A_matrix(), alg.like_B_matrix(), alg.like_B_matrix()
    L_ = lib()
    for bad in (-0.5, 1.0, math.nan, math.inf):
        assert L_.hnhd_alg_sparse_attention_dropout(alg.h, Q.h, K.h, V.h, Z.h, Lm.h, 1, 0.5, bad, 0) == -1
        assert b"dropout probability" in L_.hnh_last_error_string()
        assert L_.hnhd_alg_sparse_attention_backward_dropout(alg.h, Q.h, K.h, V.h, Z.h, Lm.h, Z.h, dQ.h, dK.h, dV.h, 1, 0.5,
                                                             bad, 0) == -1
        with pytest.raises(ValueError, match="must lie in"):
            alg.sparse_attention(Q, K, V, Z, Lm, dropout=bad)
    del S, alg
