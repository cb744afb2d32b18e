"""Fused sparse attention on the GPU at p = 1: the step, finish and two gradient kernels against the fp64 model of
tests/sparse_attention_oracle.py on every width path, leading dimension, packed form and alignment, past one resident
wave, with the online-softmax state carried across two calls and bit-identical repeats; Algorithm.sparse_attention /
sparse_attention_backward on every algorithm, square and rectangular S, 1, 2 and 4 heads, against the model and the
composed public ops (scaled SDDMM, edge softmax, SpMM).  Multi-rank cases live in
tests/test_sparse_attention_multirank_gpu.py."""
import math

import numpy as np
import pytest

from distributed_sddmm_b200 import driver as D
from tests import sparse_attention_oracle as sa
from tests.mp_edge_softmax_worker import coords

pytestmark = pytest.mark.gpu
SEED = 0xC0FFEE + 21
ALGS = ["15d_fusion1", "15d_fusion2", "15d_sparse", "25d_dense_replicate", "25d_sparse_replicate"]
WIDTHS = [4, 8, 16, 32, 64, 128, 256, 7]
# the most CTAs of 256 threads an SM holds (2048 threads per SM on sm_90)
MAX_CTAS_PER_SM = 8
KERNEL_TOL = 1e-12


def rel_err(got, ref):
    fin = np.isfinite(ref)
    assert np.array_equal(fin, np.isfinite(got)) and np.array_equal(got[~fin], ref[~fin])
    return np.abs(got[fin] - ref[fin]).max(initial=0.0) / max(np.abs(ref[fin]).max(initial=0.0), 1e-300)


@pytest.fixture(scope="module")
def world():
    D.world_init("self")
    yield
    D.world_finalize()


# ---- kernels ---------------------------------------------------------------------------------------------------
def _block(rng, M, N, long_row=1500):
    """(rowStart, rows, cols) of an M x N CSR block with empty rows, rows of one entry, a row longer than 1000 entries
    (many chunks) and duplicate pairs; sorted by row."""
    r = np.concatenate([rng.integers(0, M, 6 * M), np.full(long_row, 3)])
    r = r[((r % 7) != 5) & (r != M - 1)]  # rows 5, 12, ... stay empty
    c = rng.integers(0, N, len(r))
    r = np.concatenate([r, [1, 1, 1], [M - 1]])  # a duplicate pair, and a last row of one entry
    c = np.concatenate([c, [2, 2, 2], [0]])
    order = np.argsort(r, kind="stable")
    return _csr(r[order], c[order], M)


def _csr(r, c, M):
    rowStart = np.zeros(M + 1, np.int64)
    np.add.at(rowStart, r + 1, 1)
    return np.cumsum(rowStart), r.astype(np.int64), c.astype(np.int64)


class Side:
    """Device operands of one side of a block, each a rows x width block of a row-major matrix: `packed` puts them
    side by side in one matrix (leading dimension = the sum of widths), else each has its own with `extra` spare
    columns; `shift` doubles off the allocation's (16-byte aligned) start."""

    def __init__(self, rows, parts, packed=False, extra=0, shift=0):
        import torch
        self.parts = dict(parts)
        self.rows = rows
        self.loc = {}
        self.bufs = []
        if packed:
            ld = sum(v.shape[1] for _, v in parts)
            buf = self._alloc(torch, rows, ld, shift)
            at = 0
            for name, v in parts:
                self.loc[name] = (buf, shift + at, ld)
                at += v.shape[1]
        else:
            for name, v in parts:
                ld = v.shape[1] + extra
                self.loc[name] = (self._alloc(torch, rows, ld, shift), shift, ld)
        self.reset()

    def _alloc(self, torch, rows, ld, shift):
        buf = torch.full((rows * ld + shift + 2,), float("nan"), dtype=torch.float64, device="cuda:0")
        self.bufs.append(buf)
        return buf

    def _view(self, name):
        import torch
        buf, off, ld = self.loc[name]
        return torch.as_strided(buf, (self.rows, self.parts[name].shape[1]), (ld, 1), off)

    def reset(self):
        import torch
        for name, v in self.parts.items():
            self._view(name).copy_(torch.from_numpy(np.ascontiguousarray(v)))

    def ptr(self, name):
        buf, off, ld = self.loc[name]
        return buf.data_ptr() + 8 * off, ld

    def get(self, name):
        return self._view(name).cpu().numpy()


def _ptrs(side, *names):
    out = []
    for n in names:
        out.extend(side.ptr(n))
    return out


def _forward(L, rs, ci, rows, nnz, d, scale, R, Y, st):
    D.check(L.hnh_sparse_attention_step_f64(rs, ci, rows, nnz, d, *_ptrs(R, "Q"), *_ptrs(Y, "K", "V"), scale,
                                            *_ptrs(R, "acc", "m", "s"), st))
    D.check(L.hnh_sparse_attention_finish_f64(rows, d, *_ptrs(R, "acc", "m", "s"), *_ptrs(R, "acc", "m"), st))


def _check_kernels(rowStart, rr, cc, M, N, d, rng, packed, extra, shift, scale=None, QK=None):
    """Forward (step + finish in place), grad_q on the block and grad_kv on its transpose against the model; a
    repeat of each is bit-identical.  QK: given (Q, K) instead of random ones."""
    import torch
    from distributed_sddmm_b200 import lib
    L = lib()
    st = torch.cuda.current_stream().cuda_stream
    tol = KERNEL_TOL
    scale = 1 / math.sqrt(d) if scale is None else scale
    Qv, dZv, dQ0 = (rng.uniform(-1, 1, (M, d)) for _ in range(3))
    Kv, Vv, dK0, dV0 = (rng.uniform(-1, 1, (N, d)) for _ in range(4))
    if QK is not None:
        Qv, Kv = QK
    Zw, Lw = sa.forward_np(rr, cc, M, Qv, Kv, Vv, 1, scale)
    dQw, dKw, dVw = sa.backward_np(rr, cc, M, Qv, Kv, Vv, dZv, 1, scale)
    t_np = (dZv * Zw).sum(1, keepdims=True)
    dev = lambda x: torch.from_numpy(x).to("cuda:0")  # noqa: E731
    rs, ci = dev(rowStart), dev(cc)
    # the key-side CSR: the transpose of the block
    order = np.argsort(cc, kind="stable")
    rsT, _, ciT = _csr(cc[order], rr[order], N)
    rsT, ciT = dev(rsT), dev(ciT)
    nnz = len(cc)
    zeros = lambda n, w: np.zeros((n, w))  # noqa: E731
    # forward: m starts as NaN (not read while s = 0)
    R = Side(M, [("Q", Qv), ("acc", zeros(M, d)), ("m", np.full((M, 1), np.nan)), ("s", zeros(M, 1))], packed, extra, shift)
    Y = Side(N, [("K", Kv), ("V", Vv)], packed, extra, shift)
    got = []
    for _ in range(2):
        R.reset()
        _forward(L, rs.data_ptr(), ci.data_ptr(), M, nnz, d, scale, R, Y, st)
        torch.cuda.synchronize()
        got.append((R.get("acc"), R.get("m")[:, 0]))
        assert np.array_equal(R.get("Q"), Qv)
    assert all(np.array_equal(a, b) for a, b in zip(*got)), "forward repeat differs"
    assert rel_err(got[0][0], Zw) < tol and rel_err(got[0][1], Lw[:, 0]) < tol
    # query side
    Rq = Side(M, [("Q", Qv), ("dZ", dZv), ("L", Lw), ("t", t_np), ("dQ", dQ0)], packed, extra, shift)
    got = []
    for _ in range(2):
        Rq.reset()
        D.check(L.hnh_sparse_attention_grad_q_f64(rs.data_ptr(), ci.data_ptr(), M, nnz, d, *_ptrs(Rq, "Q", "dZ", "L", "t"),
                                                  *_ptrs(Y, "K", "V"), scale, *_ptrs(Rq, "dQ"), st))
        torch.cuda.synchronize()
        got.append(Rq.get("dQ"))
    assert np.array_equal(got[0], got[1]), "grad_q repeat differs"
    assert rel_err(got[0] - dQ0, dQw) < tol
    # key side
    Rk = Side(N, [("K", Kv), ("V", Vv), ("dK", dK0), ("dV", dV0)], packed, extra, shift)
    Yq = Side(M, [("Q", Qv), ("dZ", dZv), ("L", Lw), ("t", t_np)], packed, extra, shift)
    got = []
    for _ in range(2):
        Rk.reset()
        D.check(L.hnh_sparse_attention_grad_kv_f64(rsT.data_ptr(), ciT.data_ptr(), N, nnz, d, *_ptrs(Rk, "K", "V"),
                                                   *_ptrs(Yq, "Q", "dZ", "L", "t"), scale, *_ptrs(Rk, "dK", "dV"), st))
        torch.cuda.synchronize()
        got.append((Rk.get("dK"), Rk.get("dV")))
    assert all(np.array_equal(a, b) for a, b in zip(*got)), "grad_kv repeat differs"
    assert rel_err(got[0][0] - dK0, dKw) < tol and rel_err(got[0][1] - dV0, dVw) < tol


@pytest.mark.parametrize("d", WIDTHS)
def test_kernels_match_the_model_on_every_width(world, d):
    """Every width path (4..256 and 7 through the generic kernels), M != N, rows longer than one chunk, empty rows,
    duplicates; separate operands at leading dimension d and d + 2, the packed forms, and operands one double off
    16-byte alignment (the generic kernels)."""
    rng = np.random.default_rng(SEED + d)
    M, N = 301, 257
    rowStart, rr, cc = _block(rng, M, N)
    lens = np.diff(rowStart)
    assert (lens == 0).any() and (lens == 1).any() and lens.max() > 1000
    assert len(set(zip(rr.tolist(), cc.tolist()))) < len(rr)
    for packed, extra, shift in ((False, 0, 0), (False, 2, 0), (True, 0, 0), (False, 0, 1)):
        _check_kernels(rowStart, rr, cc, M, N, d, rng, packed, extra, shift)


@pytest.mark.parametrize("d", WIDTHS)
def test_kernels_shift_by_the_true_maximum_on_large_scores(world, d):
    """Rows whose scores all lie near -800 (or all near +800), of every length from 1 to 40: neither a multiple of the
    rows kept in flight nor of the lanes per row, so most chunks end part-full.  exp(-800) underflows, so the online
    softmax is right only if every chunk is shifted by the maximum of its own entries.  The scores are exact in fp64
    (q = +-100 (1, .., 1), <q, k_v> = +-100 d (8 + j/64), scale a power of two), so kernel and model see the same x
    and the usual bound holds."""
    rng = np.random.default_rng(SEED + 300 + d)
    M, N = 164, 64
    lens = np.arange(M) % 41  # 0 .. 40 entries
    rowStart = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    rr = np.repeat(np.arange(M), lens).astype(np.int64)
    cc = rng.integers(0, N, len(rr)).astype(np.int64)
    sign = np.where(np.arange(M) % 2 == 0, -1.0, 1.0)
    Qv = (sign * 100.0)[:, None] * np.ones((1, d))
    # k_v = a_v (1, .., 1) + w_v with w_v orthogonal to (1, .., 1): the scores depend on a_v only, and w_v keeps dQ
    # well conditioned (with K_v all close to one vector, dQ = scale sum alpha (g - t) (K_v - mean) would cancel)
    w = np.zeros((N, d))
    for i in range(d // 2):
        r = ((np.arange(N) + i) % 7 - 3).astype(np.float64)
        w[:, 2 * i], w[:, 2 * i + 1] = r, -r
    Kv = (8.0 + (np.arange(N) % 8) / 64.0)[:, None] + w
    scale = 2.0 ** -math.floor(math.log2(d))
    x = scale * (Qv[rr] * Kv[cc]).sum(1)
    assert (np.abs(x) > 745).all()  # past exp's underflow
    for packed, shift in ((False, 0), (True, 0), (False, 1)):
        _check_kernels(rowStart, rr, cc, M, N, d, rng, packed, 0, shift, scale=scale, QK=(Qv, Kv))


def test_empty_blocks_are_no_ops(world):
    import torch
    from distributed_sddmm_b200 import lib
    L = lib()
    st = torch.cuda.current_stream().cuda_stream
    x = torch.full((64,), 7.0, dtype=torch.float64, device="cuda:0")
    rs = torch.zeros(5, dtype=torch.int64, device="cuda:0")
    p, r = x.data_ptr(), rs.data_ptr()
    # four rows without entries: nothing is written
    D.check(L.hnh_sparse_attention_step_f64(r, r, 4, 0, 4, p, 4, p, 4, p, 4, 0.5, p, 4, p, 1, p, 1, st))
    D.check(L.hnh_sparse_attention_grad_q_f64(r, r, 4, 0, 4, p, 4, p, 4, p, 1, p, 1, p, 4, p, 4, 0.5, p, 4, st))
    D.check(L.hnh_sparse_attention_grad_kv_f64(r, r, 4, 0, 4, p, 4, p, 4, p, 4, p, 4, p, 1, p, 1, 0.5, p, 4, p, 4, st))
    # rows with entries but none in this block are not touched either
    rs4 = torch.tensor([0, 0, 0, 0, 0], dtype=torch.int64, device="cuda:0")
    D.check(L.hnh_sparse_attention_step_f64(rs4.data_ptr(), r, 4, 1, 4, p, 4, p, 4, p, 4, 0.5, p, 4, p, 1, p, 1, st))
    torch.cuda.synchronize()
    assert bool((x == 7.0).all())


@pytest.mark.parametrize("d", [8, 128, 7])
def test_state_carries_across_two_calls(world, d):
    """One block fed as two column-split calls (its entries with v < N/2, then the rest) equals one call."""
    import torch
    from distributed_sddmm_b200 import lib
    L = lib()
    st = torch.cuda.current_stream().cuda_stream
    rng = np.random.default_rng(SEED + 200 + d)
    M, N = 301, 257
    rowStart, rr, cc = _block(rng, M, N)
    Qv = rng.uniform(-1, 1, (M, d))
    Kv, Vv = rng.uniform(-1, 1, (N, d)), rng.uniform(-1, 1, (N, d))
    Y = Side(N, [("K", Kv), ("V", Vv)])
    dev = lambda x: torch.from_numpy(x).to("cuda:0")  # noqa: E731
    scale = 1 / math.sqrt(d)

    def state():
        return Side(M, [("Q", Qv), ("acc", np.zeros((M, d))), ("m", np.full((M, 1), np.nan)), ("s", np.zeros((M, 1)))])

    one = state()
    rs, ci = dev(rowStart), dev(cc)
    _forward(L, rs.data_ptr(), ci.data_ptr(), M, len(cc), d, scale, one, Y, st)
    two = state()
    halves = []
    for keep in (cc < N // 2, cc >= N // 2):
        r2, _, c2 = _csr(rr[keep], cc[keep], M)
        halves.append((dev(r2), dev(c2), int(keep.sum())))
    for rs2, ci2, n2 in halves:
        D.check(L.hnh_sparse_attention_step_f64(rs2.data_ptr(), ci2.data_ptr(), M, n2, d, *_ptrs(two, "Q"), *_ptrs(Y, "K", "V"),
                                                scale, *_ptrs(two, "acc", "m", "s"), st))
    D.check(L.hnh_sparse_attention_finish_f64(M, d, *_ptrs(two, "acc", "m", "s"), *_ptrs(two, "acc", "m"), st))
    torch.cuda.synchronize()
    assert rel_err(two.get("acc"), one.get("acc")) < 1e-14
    assert rel_err(two.get("m"), one.get("m")) < 1e-14


@pytest.mark.parametrize("d", [4, 64, 7])
def test_kernels_past_one_resident_wave(world, d):
    """Enough rows that every CTA of a grid capped at the resident CTAs runs at least 3 grid-stride iterations."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rows_per_cta = 256 // {4: 2, 64: 32}.get(d, 32)  # lanes per row: the width table, 32 for the generic kernels
    M = 3 * MAX_CTAS_PER_SM * sms * rows_per_cta + 5
    assert M // (MAX_CTAS_PER_SM * sms * rows_per_cta) >= 3
    rng = np.random.default_rng(SEED + 100 + d)
    N = M  # the key-side pass walks N rows
    lens = rng.integers(0, 4, M)
    rowStart = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    rr = np.repeat(np.arange(M), lens)
    cc = rng.integers(0, N, len(rr)).astype(np.int64)
    _check_kernels(rowStart, rr, cc, M, N, d, rng, False, 0, 0)


# ---- Algorithm.sparse_attention / sparse_attention_backward at p = 1 -------------------------------------------------
def _algorithm(name, shape, r):
    if shape == "square":
        S = D.SpmatLocal.load_er(7, 6, SEED)
    else:  # 150 x 97 with empty rows and duplicate pairs
        rng = np.random.default_rng(SEED + 7)
        rows = rng.integers(0, 150, 700)
        rows = rows[rows % 9 != 4]
        cols = rng.integers(0, 97, len(rows))
        rows, cols = np.concatenate([rows, [2, 2]]), np.concatenate([cols, [5, 5]])
        S = D.SpmatLocal.from_tuples(150, 97, rows, cols, np.ones(len(rows)))
    return S, D.Algorithm(name, S, r, 1)


def _dense(alg, which, values):
    m = alg.like_A_matrix() if which == "A" else alg.like_B_matrix()
    m.from_host(values)
    return m


@pytest.mark.parametrize("shape", ["square", "rectangular"])
@pytest.mark.parametrize("name", ALGS)
def test_p1_algorithm_all_algorithms(world, name, shape):
    for heads in (1, 2, 4):
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
        Zw, Lw = sa.forward_np(rows, cols, Ma, Qv, Kv, Vv, heads, scale)
        dQw, dKw, dVw = sa.backward_np(rows, cols, Ma, Qv, Kv, Vv, dZv, heads, scale)
        first = None
        for _ in range(2):
            alg.sparse_attention(Q, K, V, Z, Lm, heads)
            alg.sparse_attention_backward(Q, K, V, Z, Lm, dZ, dQ, dK, dV, heads)
            got = tuple(m.to_host() for m in (Z, Lm, dQ, dK, dV))
            if first is not None:
                assert all(np.array_equal(a, b) for a, b in zip(got, first)), (name, shape, heads)
            first = got
        where = (name, shape, heads)
        if shape == "rectangular":
            assert np.isneginf(first[1]).any(), where  # rows without entries
        for g, w in zip(first, (Zw, Lw, dQw, dKw, dVw)):
            assert rel_err(g, w) < 1e-10, where
        if heads == 1:
            # the composed public ops: scaled SDDMM, edge softmax, SpMM
            x = alg.like_S_values(0.0)
            alg.sddmmA(Q, K, alg.like_S_values(scale), x)
            alg.edge_softmax(x, "A")
            Zc = alg.like_A_matrix()
            alg.spmmA(Zc, V, x)
            assert rel_err(first[0], Zc.to_host()) < 1e-12, where
        del S, alg


def test_p1_large_scores_and_validation(world):
    """Scores of +-1000 give finite output; bad shapes, widths, head counts, scales and layouts of L are refused."""
    from distributed_sddmm_b200 import lib
    d = 8
    S, alg = _algorithm("15d_fusion2", "square", d)
    dims = alg.dims
    rng = np.random.default_rng(SEED + 9)
    # scale <q, k> = +-1000 or +-500
    Qv = rng.choice([-1.0, 1.0], (dims.localArows, 1)) * np.full((1, d), 1000 / math.sqrt(d))
    Kv = rng.choice([1.0, 0.5], (dims.localBrows, 1)) * np.ones((1, d))
    Q, K, V = _dense(alg, "A", Qv), _dense(alg, "B", Kv), _dense(alg, "B", rng.uniform(-1, 1, (dims.localBrows, d)))
    assert np.abs(Qv @ Kv.T / math.sqrt(d)).max() >= 999
    Z, Lm = alg.like_A_matrix(), D.Dense.create(dims.localArows, 1)
    dQ, dK, dV = alg.like_A_matrix(), alg.like_B_matrix(), alg.like_B_matrix()
    alg.sparse_attention(Q, K, V, Z, Lm)
    alg.sparse_attention_backward(Q, K, V, Z, Lm, alg.like_A_matrix(1.0), dQ, dK, dV)
    for m in (Z, dQ, dK, dV):
        assert np.isfinite(m.to_host()).all()
    rows, cols = coords(alg, "A")
    Zw, _ = sa.forward_np(rows, cols, dims.localArows, Qv, Kv, V.to_host(), 1, 1 / math.sqrt(d))
    assert rel_err(Z.to_host(), Zw) < 1e-10
    L_ = lib()
    bad = [
        (Q, K, V, Z, D.Dense.create(dims.localArows, 2), 1, 0.5),  # L too wide
        (Q, K, V, Z, D.Dense.create(dims.localArows + 1, 1), 1, 0.5),  # L too tall
        (Q, K, V, Z, Lm, 3, 0.5),  # 3 heads do not divide 8
        (Q, K, V, Z, Lm, 0, 0.5),
        (Q, K, V, Z, Lm, 1, math.inf),
        (Q, K, V, Z, Lm, 1, math.nan),
        (Q, K, V, D.Dense.create(dims.localArows, d - 1), Lm, 1, 0.5),  # Z too narrow
    ]
    for Qb, Kb, Vb, Zb, Lb, heads, scale in bad:
        assert L_.hnhd_alg_sparse_attention(alg.h, Qb.h, Kb.h, Vb.h, Zb.h, Lb.h, heads, scale) == -1
        assert L_.hnhd_alg_sparse_attention_backward(alg.h, Qb.h, Kb.h, Vb.h, Zb.h, Lb.h, Z.h, dQ.h, dK.h, dV.h, heads,
                                                     scale) == -1
    with pytest.raises(RuntimeError, match="code -1"):
        alg.sparse_attention_backward(Q, K, V, Z, Lm, Z, dQ, D.Dense.create(dims.localBrows, d + 1), dV)  # dK too wide
    with pytest.raises(ValueError, match="must divide"):
        alg.sparse_attention(Q, K, V, Z, Lm, heads=3)
    del S, alg
