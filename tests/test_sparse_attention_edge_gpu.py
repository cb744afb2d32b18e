"""Edge features in fused sparse attention on the GPU at p = 1: the three edge kernels against the fp64 model of
tests/sparse_attention_edge_oracle.py on every width path, with padded, packed and misaligned operands and an E with a
padded, an odd and a misaligned leading dimension, with and without dropout and bias (masked entries, rows and
chunks), past one resident wave and with the online-softmax state carried across two calls; dE checked; E = 0
bit-identical to the kernels without E.  Algorithm.sparse_attention / sparse_attention_backward with E built from
entry_coordinates on every algorithm.  Multi-rank cases live in tests/test_sparse_attention_edge_multirank_gpu.py."""
import math

import numpy as np
import pytest

from distributed_sddmm_b200 import driver as D
from tests import sparse_attention_edge_oracle as se
from tests.kernel_waves_worker import CTAS_PER_SM
from tests.test_sparse_attention_bias_gpu import _masked_bias
from tests.test_sparse_attention_gpu import ALGS, WIDTHS, Side, _algorithm, _block, _csr, _dense, _ptrs, rel_err

pytestmark = pytest.mark.gpu
SEED = 0xC0FFEE + 47
KERNEL_TOL = 1e-12
U0, V0 = 3_000_000_000, 2_500_000_123
# (packed, extra, shift) of the dense operands, and (extra, shift) of E and dE: lde = d, lde > d, odd lde, misaligned
LAYOUTS = (((False, 0, 0), (0, 0)), ((False, 2, 0), (2, 0)), ((True, 0, 0), (1, 0)), ((False, 0, 1), (0, 1)))


@pytest.fixture(scope="module")
def world():
    D.world_init("self")
    yield
    D.world_finalize()


def _rows(torch, values, extra, shift):
    """values (n x d) in a fresh NaN-filled buffer with leading dimension d + extra, `shift` doubles off its start:
    (view, pointer, ld)."""
    n, d = values.shape
    ld = d + extra
    buf = torch.full((n * ld + shift + 2,), float("nan"), dtype=torch.float64, device="cuda:0")
    view = torch.as_strided(buf, (n, d), (ld, 1), shift)
    view.copy_(torch.from_numpy(np.ascontiguousarray(values)))
    return view, buf.data_ptr() + 8 * shift, ld


def _run(L, st, dev, rs, ci, rsT, ciT, order, M, N, nnz, d, scale, Qv, Kv, Vv, dZv, dQ0, dK0, dV0, Lw, t_np, layout, drop,
         bias, E):
    """Forward (step + finish), grad_q on the block and grad_kv on its transpose, through the edge entry points (E not
    None) or the ones without E (bias None and p = 0: the plain ones; bias None: dropout; else bias).  Returns Z, L,
    dQ - dQ0, dK - dK0, dV - dV0, then dbias_A - 1 and dbias_B - 1 with a bias, then dE with E."""
    import torch
    (packed, extra, shift), (e_extra, e_shift) = layout
    p = drop[0]
    if bias is not None:
        bA, bB = dev(np.ascontiguousarray(bias)), dev(np.ascontiguousarray(bias[order]))
        dbA, dbB = dev(np.ones(nnz)), dev(np.ones(nnz))
    if E is not None:
        eA, eA_p, lde = _rows(torch, E, e_extra, e_shift)
        eB, eB_p, ldeB = _rows(torch, E[order], e_extra, e_shift)
        dE, dE_p, ldde = _rows(torch, np.full_like(E, np.nan), e_extra, e_shift)
        bq = (bA.data_ptr(), dbA.data_ptr()) if bias is not None else (None, None)
        bkv = (bB.data_ptr(), dbB.data_ptr()) if bias is not None else (None, None)
        tail = (*drop, bq[0], eA_p, lde)
        tail_q = (*drop, *bq, eA_p, lde, dE_p, ldde)
        tail_kv = (*drop, *bkv, eB_p, ldeB)
        sfx = "_edge_f64"
    elif bias is not None:
        tail, tail_q, tail_kv = (*drop, bA.data_ptr()), (*drop, bA.data_ptr(), dbA.data_ptr()), \
            (*drop, bB.data_ptr(), dbB.data_ptr())
        sfx = "_bias_f64"
    else:
        tail = tail_q = tail_kv = () if p == 0.0 else tuple(drop)
        sfx = "_f64" if p == 0.0 else "_dropout_f64"
    fn = lambda name: getattr(L, "hnh_sparse_attention_" + name + sfx)  # noqa: E731
    R = Side(M, [("Q", Qv), ("acc", np.zeros((M, d))), ("m", np.full((M, 1), np.nan)), ("s", np.zeros((M, 1)))], packed,
             extra, shift)
    Y = Side(N, [("K", Kv), ("V", Vv)], packed, extra, shift)
    D.check(fn("step")(rs, ci, M, nnz, d, *_ptrs(R, "Q"), *_ptrs(Y, "K", "V"), scale, *_ptrs(R, "acc", "m", "s"), *tail, st))
    D.check(L.hnh_sparse_attention_finish_f64(M, d, *_ptrs(R, "acc", "m", "s"), *_ptrs(R, "acc", "m"), st))
    Rq = Side(M, [("Q", Qv), ("dZ", dZv), ("L", Lw), ("t", t_np), ("dQ", dQ0)], packed, extra, shift)
    D.check(fn("grad_q")(rs, ci, M, nnz, d, *_ptrs(Rq, "Q", "dZ", "L", "t"), *_ptrs(Y, "K", "V"), scale, *_ptrs(Rq, "dQ"),
                         *tail_q, st))
    Rk = Side(N, [("K", Kv), ("V", Vv), ("dK", dK0), ("dV", dV0)], packed, extra, shift)
    Yq = Side(M, [("Q", Qv), ("dZ", dZv), ("L", Lw), ("t", t_np)], packed, extra, shift)
    D.check(fn("grad_kv")(rsT, ciT, N, nnz, d, *_ptrs(Rk, "K", "V"), *_ptrs(Yq, "Q", "dZ", "L", "t"), scale,
                          *_ptrs(Rk, "dK", "dV"), *tail_kv, st))
    torch.cuda.synchronize()
    out = (R.get("acc"), R.get("m")[:, 0], Rq.get("dQ") - dQ0, Rk.get("dK") - dK0, Rk.get("dV") - dV0)
    if bias is not None:
        out += (dbA.cpu().numpy() - 1.0, dbB.cpu().numpy() - 1.0)
    if E is not None:
        out += (dE.cpu().numpy(),)
    return out


def _check(rowStart, rr, cc, M, N, d, rng, layouts, bias, p, E=None, seed=SEED, u0=U0, v0=V0):
    """The edge kernels against the model on every layout; with E = 0 also bit-identical to the kernels without E."""
    import torch
    from distributed_sddmm_b200 import lib
    L = lib()
    st = torch.cuda.current_stream().cuda_stream
    scale = 1 / math.sqrt(d)
    nnz = len(cc)
    Qv, dZv, dQ0 = (rng.uniform(-1, 1, (M, d)) for _ in range(3))
    Kv, Vv, dK0, dV0 = (rng.uniform(-1, 1, (N, d)) for _ in range(4))
    if E is None:
        E = rng.uniform(-1, 1, (nnz, d))
    Zw, Lw = se.forward_np(rr, cc, M, Qv, Kv, Vv, E, 1, scale, p, seed, u0, v0, bias=bias)
    dQw, dKw, dVw, dEw, dbw = se.backward_np(rr, cc, M, Qv, Kv, Vv, E, dZv, 1, scale, p, seed, u0, v0, bias=bias)
    t_np = (dZv * Zw).sum(1, keepdims=True)
    Lw = Lw.reshape(M, 1)
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to("cuda:0")  # noqa: E731
    order = np.argsort(cc, kind="stable")
    rsT, _, ciT = _csr(cc[order], rr[order], N)
    ptrs = [dev(x) for x in (rowStart, cc, rsT, ciT)]
    args = [x.data_ptr() for x in ptrs] + [order, M, N, nnz, d, scale, Qv, Kv, Vv, dZv, dQ0, dK0, dV0, Lw, t_np]
    want = (Zw, Lw[:, 0], dQw, dKw, dVw) + ((dbw, dbw[order]) if bias is not None else ()) + (dEw,)
    drop = (p, seed, u0, v0)
    for layout in layouts:
        got = _run(L, st, dev, *args, layout, drop, bias, E)
        for i, (g, w) in enumerate(zip(got, want)):
            assert rel_err(g, w) < KERNEL_TOL, (d, layout, p, bias is not None, i)
        if bias is not None:
            assert not got[-1][np.isneginf(bias)].any()
        if not E.any():
            old = _run(L, st, dev, *args, layout, drop, bias, None)
            for i, (g, o) in enumerate(zip(got, old)):
                assert np.array_equal(g, o, equal_nan=True), (d, layout, p, i)
    return Zw, Lw[:, 0]


@pytest.mark.parametrize("d", WIDTHS)
def test_edge_kernels_match_the_model_on_every_width(world, d):
    """Every width path (4..256 and 7 through the generic kernels), all four combinations of dropout and bias, on
    every layout of the operands and of E: rows without entries, duplicates, a row of many chunks, masked entries,
    rows masked throughout and a masked first chunk."""
    rng = np.random.default_rng(SEED + d)
    M, N = 301, 257
    rowStart, rr, cc = _block(rng, M, N)
    bias = _masked_bias(rng, rowStart, rr, M)
    for p in (0.0, 0.5):
        for b in (None, bias):
            Zw, Lw = _check(rowStart, rr, cc, M, N, d, rng, LAYOUTS if p == 0.0 else LAYOUTS[1::2], b, p)
            if b is not None:
                dead = [u for u in range(0, M, 7) if rowStart[u + 1] > rowStart[u]]
                assert dead and not Zw[dead].any() and np.isneginf(Lw[dead]).all()


@pytest.mark.parametrize("d", WIDTHS)
def test_zero_edge_is_bit_identical_to_the_kernels_without_edge(world, d):
    rng = np.random.default_rng(SEED + 50 + d)
    M, N = 301, 257
    rowStart, rr, cc = _block(rng, M, N)
    bias = _masked_bias(rng, rowStart, rr, M)
    for p in (0.0, 0.3):
        for b in (None, bias):
            # layouts on which E takes the same kernel path as the other operands
            _check(rowStart, rr, cc, M, N, d, rng, (LAYOUTS[0], LAYOUTS[3]), b, p, E=np.zeros((len(rr), d)))


@pytest.mark.parametrize("d", [4, 64, 7])
def test_edge_kernels_past_one_resident_wave(world, d):
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rows_per_cta = 256 // {4: 2, 64: 32}.get(d, 32)
    M = 3 * CTAS_PER_SM * sms * rows_per_cta + 5
    rng = np.random.default_rng(SEED + 100 + d)
    lens = rng.integers(0, 4, M)
    rowStart = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    rr = np.repeat(np.arange(M), lens)
    cc = rng.integers(0, M, len(rr)).astype(np.int64)
    bias = rng.uniform(-1, 1, len(rr))
    bias[rng.random(len(rr)) < 0.2] = -np.inf
    _check(rowStart, rr, cc, M, M, d, rng, LAYOUTS[:1], bias, 0.5, u0=0, v0=0)


@pytest.mark.parametrize("d", [8, 128, 7])
def test_edge_state_carries_across_two_calls(world, d):
    """One block fed as two step calls (its entries with v < N/2, then the rest, each with its rows of E and of the
    bias) equals the model."""
    import torch
    from distributed_sddmm_b200 import lib
    L = lib()
    st = torch.cuda.current_stream().cuda_stream
    rng = np.random.default_rng(SEED + 200 + d)
    M, N = 301, 257
    rowStart, rr, cc = _block(rng, M, N)
    bias = rng.uniform(-3, 3, len(rr))
    bias[(rr % 3 == 0) & (cc < N // 2)] = -np.inf
    E = rng.uniform(-1, 1, (len(rr), d))
    Qv, Kv, Vv = rng.uniform(-1, 1, (M, d)), rng.uniform(-1, 1, (N, d)), rng.uniform(-1, 1, (N, d))
    Y = Side(N, [("K", Kv), ("V", Vv)])
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to("cuda:0")  # noqa: E731
    scale, p = 1 / math.sqrt(d), 0.4
    S = Side(M, [("Q", Qv), ("acc", np.zeros((M, d))), ("m", np.full((M, 1), np.nan)), ("s", np.zeros((M, 1)))])
    keep_alive = []
    for half in (cc < N // 2, cc >= N // 2):
        r2, _, c2 = _csr(rr[half], cc[half], M)
        parts = [dev(r2), dev(c2), dev(bias[half]), dev(E[half])]
        keep_alive.append(parts)
        D.check(L.hnh_sparse_attention_step_edge_f64(parts[0].data_ptr(), parts[1].data_ptr(), M, int(half.sum()), d,
                                                     *_ptrs(S, "Q"), *_ptrs(Y, "K", "V"), scale, *_ptrs(S, "acc", "m", "s"),
                                                     p, SEED, U0, V0, parts[2].data_ptr(), parts[3].data_ptr(), d, st))
    D.check(L.hnh_sparse_attention_finish_f64(M, d, *_ptrs(S, "acc", "m", "s"), *_ptrs(S, "acc", "m"), st))
    torch.cuda.synchronize()
    Zw, Lw = se.forward_np(rr, cc, M, Qv, Kv, Vv, E, 1, scale, p, SEED, U0, V0, bias=bias)
    assert rel_err(S.get("acc"), Zw) < KERNEL_TOL and rel_err(S.get("m")[:, 0], Lw[:, 0]) < KERNEL_TOL


# ---- Algorithm.sparse_attention / sparse_attention_backward with edge features at p = 1 --------------------------------
def edge_of(rows, cols, r):
    """e(u, v): r columns that are a function of the global S-row and S-column only."""
    k = np.arange(r)[None, :]
    return np.cos(0.31 * rows[:, None] + 0.73 * cols[:, None] + 0.45 * k)


def _bias_of(rows, cols):
    b = np.sin(0.37 * rows + 1.3 * cols) * 2.0
    b[(rows * 7 + cols * 3) % 9 == 4] = -np.inf
    return b


@pytest.mark.parametrize("shape", ["square", "rectangular"])
@pytest.mark.parametrize("name", ALGS)
def test_p1_algorithm_with_edge_features(world, name, shape):
    """Every algorithm, 1 and 2 heads, with and without a (shared, masked) bias, dropout 0 and 0.3: Z, L, dQ, dK, dV,
    dE (and dbias) against the model within 1e-10; a repeat is bit-identical; E = 0 equals the call without E bit for
    bit."""
    for heads in (1, 2):
        d = 4
        r = heads * d
        S, alg = _algorithm(name, shape, r)
        dims = alg.dims
        Ma, Nb = dims.localArows, dims.localBrows
        rA, cA = alg.entry_coordinates("A")
        rB, cB = alg.entry_coordinates("B")
        rng = np.random.default_rng(SEED + heads)
        Qv, dZv = rng.uniform(-1, 1, (Ma, r)), rng.uniform(-1, 1, (Ma, r))
        Kv, Vv = rng.uniform(-1, 1, (Nb, r)), rng.uniform(-1, 1, (Nb, r))
        Q, K, V, dZ = _dense(alg, "A", Qv), _dense(alg, "B", Kv), _dense(alg, "B", Vv), _dense(alg, "A", dZv)
        Z, Lm = alg.like_A_matrix(np.nan), D.Dense.create(Ma, heads, np.nan)
        dQ, dK, dV = alg.like_A_matrix(np.nan), alg.like_B_matrix(np.nan), alg.like_B_matrix(np.nan)
        scale = 1 / math.sqrt(d)

        def dense(x):
            m = D.Dense.create(*x.shape, np.nan)
            m.from_host(x)
            return m

        def vec(x):
            v = D.Vec.create(len(x), np.nan)
            v.from_host(x)
            return v

        def run(eA=None, eB=None, bA=None, bB=None, **kw):
            alg.sparse_attention(Q, K, V, Z, Lm, heads, bias=bA, edge=eA, **kw)
            dE = D.Dense.create(1, 1, np.nan) if eA is not None else None
            dbA = D.Vec.create(1, np.nan) if bA is not None else None
            alg.sparse_attention_backward(Q, K, V, Z, Lm, dZ, dQ, dK, dV, heads, bias=bA, bias_B=bB, dbias=dbA, edge=eA,
                                          edge_B=eB, dedge=dE, **kw)
            out = tuple(m.to_host() for m in (Z, Lm, dQ, dK, dV))
            return out + ((dE.to_host(),) if eA is not None else ()) + ((dbA.to_host(),) if bA is not None else ())

        EA, EB = edge_of(rA, cA, r), edge_of(rB, cB, r)
        bA, bB = _bias_of(rA, cA), _bias_of(rB, cB)
        for with_bias in (False, True):
            for p in (0.0, 0.3):
                seed = 700 + heads
                b = bA if with_bias else None
                Zw, Lw = se.forward_np(rA, cA, Ma, Qv, Kv, Vv, EA, heads, scale, p, seed, bias=b)
                dQw, dKw, dVw, dEw, dbw = se.backward_np(rA, cA, Ma, Qv, Kv, Vv, EA, dZv, heads, scale, p, seed, bias=b)
                bias_args = (vec(bA), vec(bB)) if with_bias else ()
                got = run(dense(EA), dense(EB), *bias_args, dropout=p, seed=seed)
                where = (name, shape, heads, with_bias, p)
                for g, w in zip(got, (Zw, Lw, dQw, dKw, dVw, dEw) + ((dbw,) if with_bias else ())):
                    assert rel_err(g, w) < 1e-10, where
                again = run(dense(EA), dense(EB), *((vec(bA), vec(bB)) if with_bias else ()), dropout=p, seed=seed)
                assert all(np.array_equal(a, b_) for a, b_ in zip(got, again)), where
                zero = run(dense(np.zeros_like(EA)), dense(np.zeros_like(EB)),
                           *((vec(bA), vec(bB)) if with_bias else ()), dropout=p, seed=seed)
                plain = run(None, None, *((vec(bA), vec(bB)) if with_bias else ()), dropout=p, seed=seed)
                assert all(np.array_equal(a, b_) for a, b_ in zip(zero[:5], plain[:5])), where
        del S, alg


def test_p1_edge_validation(world):
    """An E of the wrong shape, only one of edge / edge_B, a dedge without E or that is another operand: HNH_E_INVALID
    from the driver before any launch, on the forward and the backward."""
    from distributed_sddmm_b200 import lib
    heads, d = 2, 4
    r = heads * d
    S, alg = _algorithm("15d_fusion2", "square", r)
    dims = alg.dims
    Q, K, V = alg.like_A_matrix(0.5), alg.like_B_matrix(0.5), alg.like_B_matrix(0.5)
    Z, Lm = alg.like_A_matrix(), D.Dense.create(dims.localArows, heads)
    dQ, dK, dV = alg.like_A_matrix(), alg.like_B_matrix(), alg.like_B_matrix()
    nA, nB = len(alg.like_S_values()), len(alg.like_ST_values())
    L_ = lib()
    h = lambda m: m.h if m is not None else None  # noqa: E731

    def fwd(e):
        return L_.hnhd_alg_sparse_attention_edge(alg.h, Q.h, K.h, V.h, Z.h, Lm.h, heads, 0.5, 0.0, 0, None, h(e))

    def bwd(eA, eB, dE=None):
        return L_.hnhd_alg_sparse_attention_backward_edge(alg.h, Q.h, K.h, V.h, Z.h, Lm.h, Z.h, dQ.h, dK.h, dV.h, heads, 0.5,
                                                          0.0, 0, None, None, None, None, h(eA), h(eB), h(dE))

    for rows, cols in ((nA - 1, r), (nA + 1, r), (nA, r - 1), (nA, d)):
        assert fwd(D.Dense.create(rows, cols)) == -1
        assert b"its order has" in L_.hnh_last_error_string()
    EA, EB = D.Dense.create(nA, r, 0.1), D.Dense.create(nB, r, 0.1)
    assert fwd(EA) == 0 and fwd(None) == 0
    assert bwd(EA, None) == -1 and b"both orders" in L_.hnh_last_error_string()
    assert bwd(None, EB) == -1
    assert bwd(None, None, D.Dense.create(1, 1)) == -1 and b"without edge features" in L_.hnh_last_error_string()
    for alias in (EA, EB, Q, dQ, dK, dV, Z):
        assert bwd(EA, EB, alias) == -1 and b"another operand" in L_.hnh_last_error_string()
    assert bwd(EA, D.Dense.create(nB + 1, r)) == -1 and b"edge_B" in L_.hnh_last_error_string()
    dE = D.Dense.create(1, 1)
    assert bwd(EA, EB, dE) == 0 and dE.shape == (nA, r)
    assert bwd(EA, EB) == 0
    del S, alg
