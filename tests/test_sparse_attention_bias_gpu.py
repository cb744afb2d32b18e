"""Additive score bias in fused sparse attention on the GPU at p = 1: the three bias kernels against the fp64 model of
tests/sparse_attention_bias_oracle.py on every width path, leading dimension, packed form and alignment, with and
without dropout, with masked (-inf) entries, rows and chunks and biases of +-800, past one resident wave and with the
online-softmax state carried across two calls; dbias in both value orders; a bias of zeros is bit-identical to the
kernels without bias.  Algorithm.sparse_attention / sparse_attention_backward with a per-head or shared bias on every
algorithm, built from entry_coordinates, against the model and the composed public ops.  Multi-rank cases live in
tests/test_sparse_attention_bias_multirank_gpu.py."""
import math

import numpy as np
import pytest

from distributed_sddmm_b200 import driver as D
from tests import sparse_attention_bias_oracle as sb
from tests import sparse_attention_dropout_oracle as sd
from tests.kernel_waves_worker import CTAS_PER_SM
from tests.mp_edge_softmax_worker import coords
from tests.test_sparse_attention_gpu import ALGS, WIDTHS, Side, _algorithm, _block, _csr, _dense, _ptrs, rel_err

pytestmark = pytest.mark.gpu
SEED = 0xC0FFEE + 41
KERNEL_TOL = 1e-12
U0, V0 = 3_000_000_000, 2_500_000_123
LAYOUTS = ((False, 0, 0), (False, 2, 0), (True, 0, 0), (False, 0, 1))


@pytest.fixture(scope="module")
def world():
    D.world_init("self")
    yield
    D.world_finalize()


def _run(L, st, dev, rs, ci, rsT, ciT, order, M, N, nnz, d, scale, Qv, Kv, Vv, dZv, dQ0, dK0, dV0, Lw, t_np, layout, drop,
         bias):
    """Forward (step + finish), grad_q on the block and grad_kv on its transpose.  bias None: the entry points without
    bias (drop None: without dropout either); else the bias entry points with drop = (p, seed, u0, v0) and bias in the
    block's (A) order, its B-order copy bias[order].  Returns Z, L, dQ - dQ0, dK - dK0, dV - dV0, dbias_A - 1,
    dbias_B - 1 (the dbias buffers start at 1: the kernels add)."""
    import torch
    packed, extra, shift = layout
    zeros = lambda n, w: np.zeros((n, w))  # noqa: E731
    if bias is None:
        tail, tail_g = (() if drop is None else tuple(drop)), (() if drop is None else tuple(drop))
        sfx = "_f64" if drop is None else "_dropout_f64"
        dbA = dbB = None
    else:
        bA, bB = dev(np.ascontiguousarray(bias)), dev(np.ascontiguousarray(bias[order]))
        dbA, dbB = dev(np.ones(nnz)), dev(np.ones(nnz))
        tail = (*drop, bA.data_ptr())
        sfx = "_bias_f64"
    fn = lambda name: getattr(L, "hnh_sparse_attention_" + name + sfx)  # noqa: E731
    R = Side(M, [("Q", Qv), ("acc", zeros(M, d)), ("m", np.full((M, 1), np.nan)), ("s", zeros(M, 1))], packed, extra, shift)
    Y = Side(N, [("K", Kv), ("V", Vv)], packed, extra, shift)
    D.check(fn("step")(rs, ci, M, nnz, d, *_ptrs(R, "Q"), *_ptrs(Y, "K", "V"), scale, *_ptrs(R, "acc", "m", "s"), *tail, st))
    D.check(L.hnh_sparse_attention_finish_f64(M, d, *_ptrs(R, "acc", "m", "s"), *_ptrs(R, "acc", "m"), st))
    Rq = Side(M, [("Q", Qv), ("dZ", dZv), ("L", Lw), ("t", t_np), ("dQ", dQ0)], packed, extra, shift)
    gq = (*drop, bA.data_ptr(), dbA.data_ptr()) if bias is not None else tail_g
    D.check(fn("grad_q")(rs, ci, M, nnz, d, *_ptrs(Rq, "Q", "dZ", "L", "t"), *_ptrs(Y, "K", "V"), scale, *_ptrs(Rq, "dQ"),
                         *gq, st))
    Rk = Side(N, [("K", Kv), ("V", Vv), ("dK", dK0), ("dV", dV0)], packed, extra, shift)
    Yq = Side(M, [("Q", Qv), ("dZ", dZv), ("L", Lw), ("t", t_np)], packed, extra, shift)
    gkv = (*drop, bB.data_ptr(), dbB.data_ptr()) if bias is not None else tail_g
    D.check(fn("grad_kv")(rsT, ciT, N, nnz, d, *_ptrs(Rk, "K", "V"), *_ptrs(Yq, "Q", "dZ", "L", "t"), scale,
                          *_ptrs(Rk, "dK", "dV"), *gkv, st))
    torch.cuda.synchronize()
    out = (R.get("acc"), R.get("m")[:, 0], Rq.get("dQ") - dQ0, Rk.get("dK") - dK0, Rk.get("dV") - dV0)
    if bias is None:
        return out
    return out + (dbA.cpu().numpy() - 1.0, dbB.cpu().numpy() - 1.0)


def _check(rowStart, rr, cc, M, N, d, rng, layouts, bias, p, seed=SEED, scale=None, QK=None, u0=U0, v0=V0):
    """The bias kernels against the model on every layout (packed, extra, shift), dbias in both orders; a bias of zeros
    also bit-identical to the kernels without bias (with dropout: to the dropout kernels)."""
    import torch
    from distributed_sddmm_b200 import lib
    L = lib()
    st = torch.cuda.current_stream().cuda_stream
    scale = 1 / math.sqrt(d) if scale is None else scale
    Qv, dZv, dQ0 = (rng.uniform(-1, 1, (M, d)) for _ in range(3))
    Kv, Vv, dK0, dV0 = (rng.uniform(-1, 1, (N, d)) for _ in range(4))
    if QK is not None:
        Qv, Kv = QK
    Zw, Lw = sb.forward_np(rr, cc, M, Qv, Kv, Vv, bias, 1, scale, p, seed, u0, v0)
    dQw, dKw, dVw, dbw = sb.backward_np(rr, cc, M, Qv, Kv, Vv, dZv, bias, 1, scale, p, seed, u0, v0)
    t_np = (dZv * Zw).sum(1, keepdims=True)
    Lw = Lw.reshape(M, 1)
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to("cuda:0")  # noqa: E731
    order = np.argsort(cc, kind="stable")
    rsT, _, ciT = _csr(cc[order], rr[order], N)
    ptrs = [dev(x) for x in (rowStart, cc, rsT, ciT)]
    args = [x.data_ptr() for x in ptrs] + [order, M, N, len(cc), d, scale, Qv, Kv, Vv, dZv, dQ0, dK0, dV0, Lw, t_np]
    want = (Zw, Lw[:, 0], dQw, dKw, dVw, dbw, dbw[order])
    names = ("Z", "L", "dQ", "dK", "dV", "dbias_A", "dbias_B")
    drop = (p, seed, u0, v0)
    for layout in layouts:
        got = _run(L, st, dev, *args, layout, drop, bias)
        for g, w, name in zip(got, want, names):
            assert rel_err(g, w) < KERNEL_TOL, (d, layout, p, name)
        assert not got[5][np.isneginf(bias)].any() and not got[6][np.isneginf(bias[order])].any()
        if not bias.any():
            old = _run(L, st, dev, *args, layout, None if p == 0.0 else drop, None)
            for g, o, name in zip(got, old, names):
                assert np.array_equal(g, o, equal_nan=True), (d, layout, p, name)
    return Zw, Lw[:, 0]


def _masked_bias(rng, rowStart, rr, M, big=0.0):
    """A bias in [-2, 2] with 10% of the entries masked, every entry of rows 0, 7, 14, ... masked, the first 40 entries
    of row 3 (its first chunk and more) masked, and +-big added to alternate rows."""
    nnz = len(rr)
    b = rng.uniform(-2, 2, nnz)
    b[rng.random(nnz) < 0.1] = -np.inf
    b[rr % 7 == 0] = -np.inf
    b[rowStart[3]:rowStart[3] + 40] = -np.inf
    b += np.where(rr % 2 == 0, big, -big)
    return b


@pytest.mark.parametrize("d", WIDTHS)
def test_bias_kernels_match_the_model_on_every_width(world, d):
    """Every width path (4..256 and 7 through the generic kernels), without and with dropout, on every layout: a
    random bias with masked entries, rows masked throughout (Z = 0, L = -inf) and a masked first chunk."""
    rng = np.random.default_rng(SEED + d)
    M, N = 301, 257
    rowStart, rr, cc = _block(rng, M, N)
    bias = _masked_bias(rng, rowStart, rr, M)
    for p in (0.0, 0.5):
        Zw, Lw = _check(rowStart, rr, cc, M, N, d, rng, LAYOUTS if p == 0.0 else LAYOUTS[:2], bias, p)
        dead = [u for u in range(0, M, 7) if rowStart[u + 1] > rowStart[u]]
        assert dead and not Zw[dead].any() and np.isneginf(Lw[dead]).all()


@pytest.mark.parametrize("d", WIDTHS)
def test_zero_bias_is_bit_identical_to_the_kernels_without_bias(world, d):
    rng = np.random.default_rng(SEED + 50 + d)
    M, N = 301, 257
    rowStart, rr, cc = _block(rng, M, N)
    for p in (0.0, 0.3):
        _check(rowStart, rr, cc, M, N, d, rng, (LAYOUTS[0], LAYOUTS[3]), np.zeros(len(rr)), p)


@pytest.mark.parametrize("d", WIDTHS)
def test_bias_kernels_on_large_biases(world, d):
    """Biases of +-800 on alternate rows, rows of every length from 1 to 40 (most chunks part-full), masked entries
    among them: exact only if every chunk is shifted by the maximum of its own biased scores."""
    rng = np.random.default_rng(SEED + 300 + d)
    M, N = 164, 64
    lens = np.arange(M) % 41
    rowStart = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    rr = np.repeat(np.arange(M), lens).astype(np.int64)
    cc = rng.integers(0, N, len(rr)).astype(np.int64)
    bias = _masked_bias(rng, rowStart, rr, M, big=800.0)
    for p in (0.0, 0.3):
        _check(rowStart, rr, cc, M, N, d, rng, (LAYOUTS[0], LAYOUTS[2], LAYOUTS[3]), bias, p)


@pytest.mark.parametrize("d", [4, 64, 7])
def test_bias_kernels_past_one_resident_wave(world, d):
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
def test_bias_state_carries_across_two_calls(world, d):
    """One block fed as two step calls (its entries with v < N/2, then the rest, each with its own part of the bias)
    equals the model; the first call leaves rows whose first-half entries are all masked with s = 0."""
    import torch
    from distributed_sddmm_b200 import lib
    L = lib()
    st = torch.cuda.current_stream().cuda_stream
    rng = np.random.default_rng(SEED + 200 + d)
    M, N = 301, 257
    rowStart, rr, cc = _block(rng, M, N)
    bias = rng.uniform(-3, 3, len(rr))
    bias[(rr % 3 == 0) & (cc < N // 2)] = -np.inf
    Qv, Kv, Vv = rng.uniform(-1, 1, (M, d)), rng.uniform(-1, 1, (N, d)), rng.uniform(-1, 1, (N, d))
    Y = Side(N, [("K", Kv), ("V", Vv)])
    dev = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to("cuda:0")  # noqa: E731
    scale, p = 1 / math.sqrt(d), 0.4
    S = Side(M, [("Q", Qv), ("acc", np.zeros((M, d))), ("m", np.full((M, 1), np.nan)), ("s", np.zeros((M, 1)))])
    keep_alive = []
    for half in (cc < N // 2, cc >= N // 2):
        r2, _, c2 = _csr(rr[half], cc[half], M)
        parts = [dev(r2), dev(c2), dev(bias[half])]
        keep_alive.append(parts)
        D.check(L.hnh_sparse_attention_step_bias_f64(parts[0].data_ptr(), parts[1].data_ptr(), M, int(half.sum()), d,
                                                     *_ptrs(S, "Q"), *_ptrs(Y, "K", "V"), scale, *_ptrs(S, "acc", "m", "s"),
                                                     p, SEED, U0, V0, parts[2].data_ptr(), st))
    D.check(L.hnh_sparse_attention_finish_f64(M, d, *_ptrs(S, "acc", "m", "s"), *_ptrs(S, "acc", "m"), st))
    torch.cuda.synchronize()
    Zw, Lw = sb.forward_np(rr, cc, M, Qv, Kv, Vv, bias, 1, scale, p, SEED, U0, V0)
    assert rel_err(S.get("acc"), Zw) < KERNEL_TOL and rel_err(S.get("m")[:, 0], Lw[:, 0]) < KERNEL_TOL


# ---- Algorithm.sparse_attention / sparse_attention_backward with a bias at p = 1 ----------------------------------------
def _bias_of(rows, cols, h, masked=True):
    """b(u, v) for head h: a function of the global S-row and S-column only, -inf on about 1 in 9 pairs."""
    b = np.sin(0.37 * rows + 1.3 * cols + 0.5 * h) * 2.0
    if masked:
        b[(rows * 7 + cols * 3 + h) % 9 == 4] = -np.inf
    return b


@pytest.mark.parametrize("shape", ["square", "rectangular"])
@pytest.mark.parametrize("name", ALGS)
def test_p1_algorithm_with_bias(world, name, shape):
    """Every algorithm, 1 and 2 heads, per-head and shared bias, dropout 0 and 0.3: entry_coordinates equals the
    coords helper in both orders; Z, L, dQ, dK, dV and dbias in both orders against the model within 1e-10; a repeat is
    bit-identical; a bias of zeros equals the call without bias bit for bit; with a finite bias and one head the
    result matches the composed public ops (scaled sddmmA + bias, edge_softmax, spmmA) within 1e-13."""
    for heads in (1, 2):
        d = 4
        r = heads * d
        S, alg = _algorithm(name, shape, r)
        dims = alg.dims
        Ma, Nb = dims.localArows, dims.localBrows
        rA, cA = alg.entry_coordinates("A")
        rB, cB = alg.entry_coordinates("B")
        for got, want in zip((rA, cA, rB, cB), (*coords(alg, "A"), *coords(alg, "B"))):
            assert got.dtype == np.int64 and np.array_equal(got, want), (name, shape)
        rng = np.random.default_rng(SEED + heads)
        Qv, dZv = rng.uniform(-1, 1, (Ma, r)), rng.uniform(-1, 1, (Ma, r))
        Kv, Vv = rng.uniform(-1, 1, (Nb, r)), rng.uniform(-1, 1, (Nb, r))
        Q, K, V, dZ = _dense(alg, "A", Qv), _dense(alg, "B", Kv), _dense(alg, "B", Vv), _dense(alg, "A", dZv)
        Z, Lm = alg.like_A_matrix(np.nan), D.Dense.create(Ma, heads, np.nan)
        dQ, dK, dV = alg.like_A_matrix(np.nan), alg.like_B_matrix(np.nan), alg.like_B_matrix(np.nan)
        scale = 1 / math.sqrt(d)

        def vec(x):
            v = D.Vec.create(len(x), np.nan)
            v.from_host(x)
            return v

        def run(bA=None, bB=None, **kw):
            alg.sparse_attention(Q, K, V, Z, Lm, heads, bias=bA, **kw)
            dbA, dbB = (D.Vec.create(1, np.nan), D.Vec.create(1, np.nan)) if bA is not None else (None, None)
            alg.sparse_attention_backward(Q, K, V, Z, Lm, dZ, dQ, dK, dV, heads, bias=bA, bias_B=bB, dbias=dbA,
                                          dbias_B=dbB, **kw)
            out = tuple(m.to_host() for m in (Z, Lm, dQ, dK, dV))
            return out + ((dbA.to_host(), dbB.to_host()) if bA is not None else ())

        for shared in (False, True):
            hs = [0] if shared else range(heads)
            bA = np.concatenate([_bias_of(rA, cA, h) for h in hs])
            bB = np.concatenate([_bias_of(rB, cB, h) for h in hs])
            for p in (0.0, 0.3):
                seed = 500 + heads
                Zw, Lw = sb.forward_np(rA, cA, Ma, Qv, Kv, Vv, bA, heads, scale, p, seed)
                dQw, dKw, dVw, dbw = sb.backward_np(rA, cA, Ma, Qv, Kv, Vv, dZv, bA, heads, scale, p, seed)
                # dbias in the B order: the model's A-order gradient at the same (u, v), per head
                _, _, _, dbwB = sb.backward_np(rB, cB, Ma, Qv, Kv, Vv, dZv, bB, heads, scale, p, seed)
                got = run(vec(bA), vec(bB), dropout=p, seed=seed)
                where = (name, shape, heads, shared, p)
                for g, w in zip(got, (Zw, Lw, dQw, dKw, dVw, dbw, dbwB)):
                    assert rel_err(g, w) < 1e-10, where
                assert all(np.array_equal(a, b) for a, b in zip(got, run(vec(bA), vec(bB), dropout=p, seed=seed))), where
        zero = run(vec(np.zeros(len(rA))), vec(np.zeros(len(rB))))
        assert all(np.array_equal(a, b) for a, b in zip(zero[:5], run())), (name, shape, heads)
        if heads == 1:
            bA, bB = _bias_of(rA, cA, 0, masked=False), _bias_of(rB, cB, 0, masked=False)
            fused = run(vec(bA), vec(bB))
            x = alg.like_S_values(0.0)
            alg.sddmmA(Q, K, alg.like_S_values(scale), x)
            x.from_host(x.to_host() + bA)
            alg.edge_softmax(x, "A")
            Zc = alg.like_A_matrix()
            alg.spmmA(Zc, V, x)
            assert rel_err(fused[0], Zc.to_host()) < 1e-13, (name, shape)
        del S, alg


def test_p1_bias_validation(world):
    """Wrong bias lengths, bias_A and bias_B of different head multiplicity, only one of them, a dbias without its bias
    or aliasing a bias: HNH_E_INVALID from the driver before any launch; entry_coordinates with a bad mode."""
    from distributed_sddmm_b200 import lib
    heads, d = 2, 4
    S, alg = _algorithm("15d_fusion2", "square", heads * d)
    dims = alg.dims
    Q, K, V = alg.like_A_matrix(0.5), alg.like_B_matrix(0.5), alg.like_B_matrix(0.5)
    Z, Lm = alg.like_A_matrix(), D.Dense.create(dims.localArows, heads)
    dQ, dK, dV = alg.like_A_matrix(), alg.like_B_matrix(), alg.like_B_matrix()
    nA, nB = len(alg.like_S_values()), len(alg.like_ST_values())
    L_ = lib()

    def fwd(b):
        return L_.hnhd_alg_sparse_attention_bias(alg.h, Q.h, K.h, V.h, Z.h, Lm.h, heads, 0.5, 0.0, 0, b.h if b else None)

    def bwd(bA, bB, dA=None, dB=None):
        h = lambda v: v.h if v is not None else None  # noqa: E731
        return L_.hnhd_alg_sparse_attention_backward_bias(alg.h, Q.h, K.h, V.h, Z.h, Lm.h, Z.h, dQ.h, dK.h, dV.h, heads, 0.5,
                                                          0.0, 0, h(bA), h(bB), h(dA), h(dB))

    for bad in (nA - 1, nA + 1, 3 * nA):
        assert fwd(D.Vec.create(bad)) == -1
        assert b"entries; its order has" in L_.hnh_last_error_string()
    assert fwd(D.Vec.create(nA)) == 0 and fwd(D.Vec.create(heads * nA)) == 0
    shared_A, shared_B, per_A, per_B = D.Vec.create(nA), D.Vec.create(nB), D.Vec.create(heads * nA), D.Vec.create(heads * nB)
    assert bwd(shared_A, per_B) == -1 and b"per head" in L_.hnh_last_error_string()
    assert bwd(shared_A, None) == -1 and b"both orders" in L_.hnh_last_error_string()
    assert bwd(None, shared_B) == -1
    assert bwd(None, None, D.Vec.create(1)) == -1 and b"without its bias" in L_.hnh_last_error_string()
    assert bwd(shared_A, shared_B, shared_A) == -1 and b"may not be a bias" in L_.hnh_last_error_string()
    assert bwd(shared_A, shared_B, None, shared_A) == -1
    one = D.Vec.create(1)
    assert bwd(shared_A, shared_B, one, one) == -1
    assert bwd(shared_A, D.Vec.create(nB + 1)) == -1
    dA, dB = D.Vec.create(1), D.Vec.create(1)
    assert bwd(per_A, per_B, dA, dB) == 0 and len(dA) == heads * nA and len(dB) == heads * nB
    assert bwd(shared_A, shared_B, None, dB) == 0 and len(dB) == nB
    rows = D.Vec.create(1)
    assert L_.hnhd_alg_entry_coordinates(alg.h, 2, rows.h, D.Vec.create(1).h) == -1
    assert L_.hnhd_alg_entry_coordinates(alg.h, 0, rows.h, rows.h) == -1
    with pytest.raises(ValueError):
        alg.entry_coordinates("C")
    del S, alg
