"""Edge softmax on the GPU: the new kernels against numpy, Algorithm.edge_softmax / edge_softmax_backward at p = 1 on
every algorithm in both value orders, and softmax graph attention forward + backward at p = 1 against the autograd
model of tests/gat_softmax_oracle.py.  Multi-rank cases live in tests/test_edge_softmax_multirank_gpu.py."""
import ctypes as C

import numpy as np
import pytest

from distributed_sddmm_b200 import driver as D
from oracle import hnh_oracle as orc
from tests import gat_softmax_oracle as gso
from tests.mp_worker import gat_inputs

pytestmark = pytest.mark.gpu
SEED = 0xC0FFEE + 3
ALGS = ["15d_fusion1", "15d_fusion2", "15d_sparse", "25d_dense_replicate", "25d_sparse_replicate"]
LAYERS = [[12, 8, 2], [16, 4, 3]]
# the value vector of the A order lives in ST's blocks for these (their blocks are stored transposed)
A_IN_ST = {"15d_fusion1", "25d_dense_replicate"}


def rel_err(got, ref):
    return np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-300)


@pytest.fixture(scope="module")
def world():
    D.world_init("self")
    yield
    D.world_finalize()


# ---- kernels ---------------------------------------------------------------------------------------------------
def _plan(L, torch, dev, keys_np, M):
    st = torch.cuda.current_stream().cuda_stream
    n = len(keys_np)
    keys = torch.from_numpy(keys_np.astype(np.int32)).to(dev)
    cap = L.hnh_edge_softmax_piece_bound(n, M)
    I32 = dict(dtype=torch.int32, device=dev)
    perm, rs, pf = torch.full((max(n, 1),), -1, **I32), torch.full((M + 1,), -1, **I32), torch.full((M + 1,), -1, **I32)
    pr = torch.full((max(cap, 1),), -1, **I32)
    npieces = C.c_int64(-1)
    D.check(L.hnh_edge_softmax_plan(keys.data_ptr(), n, M, perm.data_ptr(), rs.data_ptr(), pf.data_ptr(), pr.data_ptr(), cap,
                                    C.byref(npieces), st), "plan")
    return dict(keys=keys, perm=perm, rs=rs, pf=pf, pr=pr, P=npieces.value, M=M, n=n, st=st)


def _softmax(L, torch, dev, pl, x):
    """alpha (NaN-prefilled output) and the row statistics through the kernels."""
    nan = dict(dtype=torch.float64, device=dev)
    P, M, st = pl["P"], pl["M"], pl["st"]
    pm, ps = torch.full((max(P, 1),), float("nan"), **nan), torch.full((max(P, 1),), float("nan"), **nan)
    rm, rsum = torch.full((M,), float("nan"), **nan), torch.full((M,), float("nan"), **nan)
    D.check(L.hnh_edge_softmax_stats_f64(x.data_ptr(), pl["perm"].data_ptr(), pl["rs"].data_ptr(), pl["pf"].data_ptr(),
                                         pl["pr"].data_ptr(), M, P, pm.data_ptr(), ps.data_ptr(), rm.data_ptr(), rsum.data_ptr(), st))
    a = torch.full_like(x, float("nan"))
    D.check(L.hnh_edge_softmax_apply_f64(a.data_ptr(), x.data_ptr(), pl["keys"].data_ptr(), pl["n"], rm.data_ptr(),
                                         rsum.data_ptr(), st))
    torch.cuda.synchronize()
    return a, rm, rsum


def _backward(L, torch, dev, pl, a, g):
    P, M, st = pl["P"], pl["M"], pl["st"]
    pd = torch.full((max(P, 1),), float("nan"), dtype=torch.float64, device=dev)
    rd = torch.full((M,), float("nan"), dtype=torch.float64, device=dev)
    D.check(L.hnh_edge_softmax_dot_f64(a.data_ptr(), g.data_ptr(), pl["perm"].data_ptr(), pl["rs"].data_ptr(), pl["pf"].data_ptr(),
                                       pl["pr"].data_ptr(), M, P, pd.data_ptr(), rd.data_ptr(), st))
    dx = torch.full_like(a, float("nan"))
    D.check(L.hnh_edge_softmax_backward_f64(dx.data_ptr(), a.data_ptr(), g.data_ptr(), pl["keys"].data_ptr(), pl["n"],
                                            rd.data_ptr(), st))
    torch.cuda.synchronize()
    return dx, rd


def _ragged_keys(rng):
    """Rows of ragged length in shuffled order: empty rows, one-entry rows, rows of thousands of entries (several
    pieces), and the last row."""
    M = 700
    lens = rng.integers(0, 40, M)
    lens[::7] = 0
    lens[3::11] = 1
    lens[5], lens[100], lens[101], lens[M - 1] = 5000, 2048, 1025, 3
    keys = np.repeat(np.arange(M), lens)
    rng.shuffle(keys)
    return keys, M


def test_kernels_against_numpy(world):
    import torch
    from distributed_sddmm_b200 import lib
    L = lib()
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(31)
    keys, M = _ragged_keys(rng)
    pl = _plan(L, torch, dev, keys, M)
    # the plan: perm groups the entries by key, stably; row_start delimits the rows
    perm = pl["perm"].cpu().numpy()
    assert np.array_equal(perm, np.argsort(keys, kind="stable"))
    assert np.array_equal(pl["rs"].cpu().numpy(), np.searchsorted(keys[perm], np.arange(M + 1)))
    lens = np.bincount(keys, minlength=M)
    assert pl["P"] == int(np.sum((lens + 1023) // 1024))
    for scale in (1.0, 1000.0):
        x_np = rng.uniform(-scale, scale, len(keys))
        x_np[::13] = scale  # ties with the maximum
        x = torch.from_numpy(x_np).to(dev)
        a, rm, rsum = _softmax(L, torch, dev, pl, x)
        want = gso.edge_softmax_np(x_np, keys, M)
        got = a.cpu().numpy()
        assert np.isfinite(got).all()
        assert np.abs(got - want).max() <= 1e-13 * np.abs(want).max(), scale
        # the row statistics of rows without entries are (-inf, 0); every other row sums to one
        empty = lens == 0
        assert np.all(rm.cpu().numpy()[empty] == -np.inf) and np.all(rsum.cpu().numpy()[empty] == 0)
        sums = np.zeros(M)
        np.add.at(sums, keys, got)
        assert np.abs(sums[~empty] - 1).max() < 1e-13
        # bit-identical repeat
        a2, _, _ = _softmax(L, torch, dev, pl, x)
        assert torch.equal(a, a2)
        # in place
        xi = x.clone()
        D.check(L.hnh_edge_softmax_apply_f64(xi.data_ptr(), xi.data_ptr(), pl["keys"].data_ptr(), pl["n"], rm.data_ptr(),
                                             rsum.data_ptr(), pl["st"]))
        torch.cuda.synchronize()
        assert torch.equal(xi, a)
        # backward
        g_np = rng.uniform(-1, 1, len(keys))
        g = torch.from_numpy(g_np).to(dev)
        dx, _ = _backward(L, torch, dev, pl, a, g)
        want_dx = gso.edge_softmax_backward_np(got, g_np, keys, M)
        assert np.abs(dx.cpu().numpy() - want_dx).max() <= 1e-13 * np.abs(want_dx).max()
        dx2, _ = _backward(L, torch, dev, pl, a, g)
        assert torch.equal(dx, dx2)
        gi = g.clone()
        rd = torch.zeros(M, dtype=torch.float64, device=dev)
        pd = torch.zeros(max(pl["P"], 1), dtype=torch.float64, device=dev)
        D.check(L.hnh_edge_softmax_dot_f64(a.data_ptr(), gi.data_ptr(), pl["perm"].data_ptr(), pl["rs"].data_ptr(),
                                           pl["pf"].data_ptr(), pl["pr"].data_ptr(), M, pl["P"], pd.data_ptr(), rd.data_ptr(), pl["st"]))
        D.check(L.hnh_edge_softmax_backward_f64(gi.data_ptr(), a.data_ptr(), gi.data_ptr(), pl["keys"].data_ptr(), pl["n"],
                                                rd.data_ptr(), pl["st"]))
        torch.cuda.synchronize()
        assert torch.equal(gi, dx)


def test_rescale_and_plan_errors(world):
    import torch
    from distributed_sddmm_b200 import lib
    L = lib()
    dev = torch.device("cuda:0")
    st = torch.cuda.current_stream().cuda_stream
    s = torch.tensor([2.0, 0.0, 3.0], dtype=torch.float64, device=dev)
    ml = torch.tensor([1.0, -np.inf, 5.0], dtype=torch.float64, device=dev)
    mg = torch.tensor([4.0, 7.0, 5.0], dtype=torch.float64, device=dev)
    D.check(L.hnh_edge_softmax_rescale_f64(s.data_ptr(), ml.data_ptr(), mg.data_ptr(), 3, st))
    torch.cuda.synchronize()
    assert np.allclose(s.cpu().numpy(), [2.0 * np.exp(-3.0), 0.0, 3.0], rtol=1e-15, atol=0)
    # a key outside [0, M) is refused before anything is written
    with pytest.raises(RuntimeError, match="outside"):
        _plan(L, torch, dev, np.array([0, 3, 1]), 3)
    with pytest.raises(RuntimeError, match="outside"):
        _plan(L, torch, dev, np.array([0, -1]), 3)
    # no entries: every row is empty
    pl = _plan(L, torch, dev, np.zeros(0, np.int64), 5)
    assert pl["P"] == 0 and np.array_equal(pl["rs"].cpu().numpy(), np.zeros(6))
    x = torch.zeros(0, dtype=torch.float64, device=dev)
    _, rm, rsum = _softmax(L, torch, dev, pl, x)
    assert np.all(rm.cpu().numpy() == -np.inf) and np.all(rsum.cpu().numpy() == 0)


# ---- Algorithm.edge_softmax at p = 1 ----------------------------------------------------------------------------
def _entry_coords(alg, name, mode):
    """(S-row, S-col) of every entry of a value vector of `mode`, from Algorithm.blocks(): the A order lives in S's
    blocks (ST's for fusion 1 and 2.5D dense), the B order in the other matrix's; ST holds the transposed tuples;
    a transposed block stores its tuples' columns as rows."""
    holder = ("ST" if name in A_IN_ST else "S") if mode == "A" else ("S" if name in A_IN_ST else "ST")
    blocks = alg.blocks(holder)
    assert len(blocks) == 1
    b = blocks[0]
    r, c = (b["col_idx"], b["row_idx"]) if b["transpose"] else (b["row_idx"], b["col_idx"])
    return (c, r) if holder == "ST" else (r, c)


def _coords_by_sddmm(alg, mode, N):
    """The same coordinates from two SDDMMs of index columns, independent of the block layout."""
    R = alg.dims.R
    A, B = alg.like_A_matrix(), alg.like_B_matrix()
    like = alg.like_S_values if mode == "A" else alg.like_ST_values
    sddmm = alg.sddmmA if mode == "A" else alg.sddmmB
    ones, res = like(1.0), like(0.0)
    out = []
    for first in ("A", "B"):
        a, b = np.zeros((N, R)), np.zeros((N, R))
        a[:, 0] = np.arange(N) if first == "A" else 1.0
        b[:, 0] = np.arange(N) if first == "B" else 1.0
        A.from_host(a)
        B.from_host(b)
        sddmm(A, B, ones, res)
        out.append(np.rint(res.to_host()).astype(np.int64))
    return out


def _score(r, c):
    """Deterministic edge scores over a wide range (up to +-1000)."""
    return 1000.0 * np.sin(0.37 * r + 1.91 * c) * np.cos(0.11 * c)


@pytest.mark.parametrize("name", ALGS)
def test_p1_edge_softmax_all_algorithms_both_orders(world, name):
    logM, npr, R = 8, 7, 8
    N = 1 << logM
    S = D.SpmatLocal.load_er(logM, npr, SEED)
    alg = D.Algorithm(name, S, R, 1)
    for mode in ("A", "B"):
        r, c = _entry_coords(alg, name, mode)
        r2, c2 = _coords_by_sddmm(alg, mode, N)
        assert np.array_equal(r, r2) and np.array_equal(c, c2), (name, mode)
        v = (alg.like_S_values if mode == "A" else alg.like_ST_values)(0.0)
        x = _score(r, c)
        v.from_host(x)
        alg.edge_softmax(v, mode)
        a = v.to_host()
        want = gso.edge_softmax_np(x, r, N)
        assert np.isfinite(a).all()
        assert rel_err(a, want) < 1e-13, (name, mode)
        # bit-identical repeat (the plan is cached after the first call)
        v.from_host(x)
        alg.edge_softmax(v, mode)
        assert np.array_equal(v.to_host(), a)
        # backward
        gr = np.cos(0.5 * r - 0.3 * c)
        alpha = (alg.like_S_values if mode == "A" else alg.like_ST_values)(0.0)
        alpha.from_host(a)
        g = (alg.like_S_values if mode == "A" else alg.like_ST_values)(0.0)
        g.from_host(gr)
        alg.edge_softmax_backward(alpha, g, mode)
        want_dx = gso.edge_softmax_backward_np(a, gr, r, N)
        assert rel_err(g.to_host(), want_dx) < 1e-13, (name, mode)
    # a vector of the wrong length is refused
    with pytest.raises(RuntimeError, match="code -1"):
        alg.edge_softmax(D.Vec(_vec_handle(alg.dims.s_values - 1)), "A")


def _vec_handle(n):
    from distributed_sddmm_b200 import lib
    h = C.c_void_p()
    D.check(lib().hnhd_vec_create(n, 0.0, C.byref(h)))
    return h


# ---- softmax graph attention at p = 1 -------------------------------------------------------------------------
def _p1_net(name, logM=8, npr=6):
    N = 1 << logM
    rows, cols, _ = orc.er_tuples(logM, npr, SEED)
    layers, X0, weights = gat_inputs(N, LAYERS, SEED)
    S = D.SpmatLocal.load_er(logM, npr, SEED)
    alg = D.Algorithm(name, S, layers[0][0], 1)
    net = D.GAT(alg, layers, 0.2, attention="softmax")
    for i, (_, _, heads) in enumerate(layers):
        for h in range(heads):
            net.set_weight(i, h, weights[i][h])
    net.set_input(X0)
    G = np.random.default_rng(SEED + 5).uniform(-1, 1, net.buffer_shape(len(layers)))
    return dict(N=N, rows=rows, cols=cols, layers=layers, X0=X0, weights=weights, S=S, alg=alg, net=net, G=G)


@pytest.mark.parametrize("name", ALGS)
def test_p1_softmax_gat_matches_autograd(world, name):
    P = _p1_net(name)
    net, layers = P["net"], P["layers"]
    net.forward()
    out = net.buffer(len(layers))
    want = gso.gat_softmax_forward_global(P["rows"], P["cols"], P["N"], layers, P["weights"], 0.2, P["X0"])
    assert np.abs(want).max() > 0
    assert rel_err(out, want) < 1e-10, name
    net.backward(P["G"])
    dX0, dW = gso.gat_softmax_backward_global(P["rows"], P["cols"], P["N"], layers, P["weights"], 0.2, P["X0"], P["G"])
    assert np.abs(dX0).max() > 0
    assert rel_err(net.input_grad(), dX0) < 1e-10, name
    for i, (_, _, heads) in enumerate(layers):
        for h in range(heads):
            assert np.abs(dW[i][h]).max() > 0, (i, h)
            assert rel_err(net.weight_grad(i, h), dW[i][h]) < 1e-10, (name, i, h)
    # the backward pass leaves the activations alone; a second forward pass is bit-identical
    assert np.array_equal(net.buffer(len(layers)), out)
    net.forward()
    assert np.array_equal(net.buffer(len(layers)), out)


def test_p1_attention_switch(world):
    """Switching the attention makes the activations stale; "leaky" is the default and stays the reference formula
    bit for bit; a bogus kind is refused by the C entry point too."""
    from distributed_sddmm_b200 import lib
    P = _p1_net("15d_fusion2", logM=7, npr=5)
    net, layers = P["net"], P["layers"]
    net.forward()
    soft = net.buffer(len(layers))
    net.set_attention("leaky")
    with pytest.raises(RuntimeError, match="no forward pass"):
        net.backward(P["G"])
    net.forward()
    leaky = net.buffer(len(layers))
    plain = D.GAT(P["alg"], layers, 0.2)  # default attention
    assert plain.attention == "leaky"
    for i, (_, _, heads) in enumerate(layers):
        for h in range(heads):
            plain.set_weight(i, h, P["weights"][i][h])
    plain.set_input(P["X0"])
    plain.forward()
    assert np.array_equal(plain.buffer(len(layers)), leaky)
    assert not np.allclose(soft, leaky)
    net.set_attention("softmax")
    net.forward()
    assert np.array_equal(net.buffer(len(layers)), soft)
    assert lib().hnhd_gat_set_attention(net.h, b"bogus") == -1
    assert b"attention" in lib().hnh_last_error_string()


def test_gat_softmax_benchmark_records(world):
    S = D.SpmatLocal.load_er(10, 8, SEED)
    for app in ("gat_softmax", "gat_softmax_train"):
        rec = D.benchmark_algorithm(S, "15d_fusion1", R=32, c=1, fused=True, app=app, trials=1, warmup=0)
        assert rec["overall_throughput"] > 0 and rec["elapsed"] > 0, app
