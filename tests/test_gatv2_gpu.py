"""GATv2 attention on the GPU at p = 1: the two new kernels against numpy (bit-equal on small-integer operands) on every
width path, leading dimension and alignment, past one resident wave; Algorithm.gatv2_scores / gatv2_backward on every
algorithm in both value orders; and the GATv2 GAT forward + backward (dX0, every dW, every da) and three SGD steps
against the autograd model of tests/gatv2_oracle.py.  Multi-rank cases live in tests/test_gatv2_multirank_gpu.py."""
import ctypes as C

import numpy as np
import pytest

from distributed_sddmm_b200 import driver as D
from oracle import hnh_oracle as orc
from tests import gatv2_oracle as g2
from tests.mp_edge_softmax_worker import coords
from tests.mp_worker import gat_inputs

pytestmark = pytest.mark.gpu
SEED = 0xC0FFEE + 8
ALGS = ["15d_fusion1", "15d_fusion2", "15d_sparse", "25d_dense_replicate", "25d_sparse_replicate"]
LAYERS = [[12, 8, 2], [16, 5, 3]]  # the second layer's heads are 5 wide: the generic kernels
ALPHA = 0.2
EXACT_ALPHA = 0.25  # with small-integer operands every product and sum below is exact in fp64
WIDTHS = [4, 8, 16, 32, 64, 128, 256, 7]
# the most CTAs of 256 threads an SM holds (2048 threads per SM on sm_90)
MAX_CTAS_PER_SM = 8


def rel_err(got, ref):
    return np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-300)


@pytest.fixture(scope="module")
def world():
    D.world_init("self")
    yield
    D.world_finalize()


def _vec(n, value=0.0):
    from distributed_sddmm_b200 import lib
    h = C.c_void_p()
    D.check(lib().hnhd_vec_create(n, value, C.byref(h)))
    return D.Vec(h)


# ---- kernels ---------------------------------------------------------------------------------------------------
def _block(rng, M, N, long_row=1500):
    """CSR rows of M x N with empty rows, rows of one entry, a row longer than 1000 entries, duplicate (u, v) pairs
    and self-loops; sorted by row."""
    r = np.concatenate([rng.integers(0, M, 6 * M), np.full(long_row, 3)])
    r = r[((r % 7) != 5) & (r != M - 1)]  # rows 5, 12, ... stay empty
    c = rng.integers(0, N, len(r))
    c[::11] = np.minimum(r[::11], N - 1)  # self-loops
    r = np.concatenate([r, [1, 1, 1], [M - 1]])  # a duplicate pair, and a last row of one entry
    c = np.concatenate([c, [2, 2, 2], [0]])
    order = np.argsort(r, kind="stable")
    r, c = r[order], c[order]
    rowStart = np.zeros(M + 1, np.int64)
    np.add.at(rowStart, r + 1, 1)
    return np.cumsum(rowStart), r, c.astype(np.int64)


def _dense(torch, rows, r, ld, shift, values):
    """rows x r values inside a (rows x ld) device matrix starting `shift` doubles into its allocation."""
    import torch as T
    buf = T.zeros(rows * ld + shift + 2, dtype=T.float64, device="cuda:0")
    view = buf[shift:shift + rows * ld].view(rows, ld)
    view[:, :r] = T.from_numpy(values).to("cuda:0")
    return buf, view, buf.data_ptr() + 8 * shift


def _run_kernels(L, torch, rowStart, rr, cc, M, N, r, ldr, ldy, shift, rng, packed=False):
    """scores and grad (with da) on one block; returns (out, dR, da) as numpy, after checking a repeat is identical"""
    import torch as T
    st = T.cuda.current_stream().cuda_stream
    dev = "cuda:0"
    nnz = len(cc)
    Rv = rng.integers(-3, 4, (M, r)).astype(np.float64)
    Yv = rng.integers(-3, 4, (N, r)).astype(np.float64)
    a_np = rng.integers(-2, 3, r).astype(np.float64)
    g_np = rng.integers(-2, 3, nnz).astype(np.float64)
    dR0 = rng.integers(-2, 3, (M, r)).astype(np.float64)
    if packed:  # [R | dR] as one 2r-wide matrix
        Q = np.concatenate([Rv, dR0], 1)
        qbuf, qview, qptr = _dense(torch, M, 2 * r, 2 * r, shift, Q)
        Rp, ldr_, dRp, lddr = qptr, 2 * r, qptr + 8 * r, 2 * r
        keep = [qbuf]
    else:
        rbuf, _, Rp = _dense(torch, M, r, ldr, shift, Rv)
        dbuf, dview, dRp = _dense(torch, M, r, ldr, shift, dR0)
        ldr_, lddr = ldr, ldr
        keep = [rbuf, dbuf]
    ybuf, _, Yp = _dense(torch, N, r, ldy, shift, Yv)
    abuf = T.zeros(r + 2, dtype=T.float64, device=dev)
    abuf[shift:shift + r] = T.from_numpy(a_np).to(dev)
    ap = abuf.data_ptr() + 8 * shift
    rs = T.from_numpy(rowStart).to(dev)
    ci = T.from_numpy(cc).to(dev)
    g = T.from_numpy(g_np).to(dev)
    results = []
    for _ in range(2):
        out = T.full((nnz,), float("nan"), dtype=T.float64, device=dev)
        D.check(L.hnh_gatv2_scores_f64(rs.data_ptr(), ci.data_ptr(), M, nnz, Rp, ldr_, Yp, ldy, ap, r, EXACT_ALPHA, out.data_ptr(), st))
        ws_bytes = L.hnh_gatv2_grad_workspace_bytes(M, r)
        ws = T.full((max(ws_bytes // 8, 1),), float("nan"), dtype=T.float64, device=dev)
        da = T.from_numpy(np.arange(r, dtype=np.float64)).to(dev)  # accumulated onto
        before = [k.clone() for k in keep]
        D.check(L.hnh_gatv2_grad_f64(rs.data_ptr(), ci.data_ptr(), g.data_ptr(), M, nnz, Rp, ldr_, Yp, ldy, ap, r, EXACT_ALPHA,
                                     dRp, lddr, da.data_ptr(), ws.data_ptr(), ws_bytes, st))
        T.cuda.synchronize()
        if packed:
            dR = keep[0][shift:shift + M * 2 * r].view(M, 2 * r)[:, r:].cpu().numpy()
            assert np.array_equal(keep[0][shift:shift + M * 2 * r].view(M, 2 * r)[:, :r].cpu().numpy(), Rv)  # R untouched
        else:
            dR = keep[1][shift:shift + M * ldr].view(M, ldr)[:, :r].cpu().numpy()
            assert T.equal(keep[1][shift:shift + M * ldr].view(M, ldr)[:, r:], before[1][shift:shift + M * ldr].view(M, ldr)[:, r:])
        results.append((out.cpu().numpy(), dR.copy(), da.cpu().numpy() - np.arange(r)))
        # restore the accumulated gradient for the repeat
        for k, b in zip(keep, before):
            k.copy_(b)
    assert all(np.array_equal(x, y) for x, y in zip(results[0], results[1])), "repeat differs"
    want_out = g2.scores_np(Rv, Yv, rr, cc, a_np, EXACT_ALPHA)
    dR_inc, want_da = g2.grad_np(Rv, Yv, rr, cc, g_np, a_np, EXACT_ALPHA)
    return results[0], (want_out, dR0 + dR_inc, want_da)


@pytest.mark.parametrize("r", WIDTHS)
def test_kernels_bit_equal_numpy_on_every_width(world, r):
    """Every width path (4..256 and 7 through the generic kernels), M != N, leading dimensions r, r + 2 and the 2r
    packed form, and operands one double off 16-byte alignment (the generic kernels)."""
    import torch
    from distributed_sddmm_b200 import lib
    L = lib()
    rng = np.random.default_rng(SEED + r)
    M, N = 301, 257
    rowStart, rr, cc = _block(rng, M, N)
    lens = np.diff(rowStart)
    assert (lens == 0).any() and (lens == 1).any() and lens.max() > 1000
    assert len(set(zip(rr.tolist(), cc.tolist()))) < len(rr) and (rr == cc).any()
    for ldr, ldy, shift, packed in ((r, r, 0, False), (r + 2, r + 4, 0, False), (2 * r, r, 0, True), (r, r, 1, False)):
        (out, dR, da), (w_out, w_dR, w_da) = _run_kernels(L, torch, rowStart, rr, cc, M, N, r, ldr, ldy, shift, rng, packed)
        where = (r, ldr, ldy, shift, packed)
        assert np.array_equal(out, w_out), where
        assert np.array_equal(dR, w_dR), where
        assert np.array_equal(da, w_da), where


def test_kernels_empty_blocks_are_no_ops(world):
    import torch
    from distributed_sddmm_b200 import lib
    L = lib()
    st = torch.cuda.current_stream().cuda_stream
    x = torch.full((64,), 7.0, dtype=torch.float64, device="cuda:0")
    rs = torch.zeros(5, dtype=torch.int64, device="cuda:0")
    p = x.data_ptr()
    # four rows without entries: nothing is written
    D.check(L.hnh_gatv2_scores_f64(rs.data_ptr(), rs.data_ptr(), 4, 0, p, 4, p, 4, p, 4, 0.2, p, st))
    D.check(L.hnh_gatv2_grad_f64(rs.data_ptr(), rs.data_ptr(), p, 4, 0, p, 4, p, 4, p, 4, 0.2, p, 4, p, p, 512, st))
    torch.cuda.synchronize()
    assert bool((x == 7.0).all())


@pytest.mark.parametrize("r", [4, 64, 7])
def test_kernels_past_one_resident_wave(world, r):
    """Enough rows that every CTA of a grid capped at the resident CTAs runs at least 3 grid-stride iterations."""
    import torch
    from distributed_sddmm_b200 import lib
    L = lib()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rows_per_cta = 256 // {4: 2, 64: 32}.get(r, 32)  # lanes per row: the width table, 32 for the generic kernels
    M = 3 * MAX_CTAS_PER_SM * sms * rows_per_cta + 5
    assert M // (MAX_CTAS_PER_SM * sms * rows_per_cta) >= 3
    rng = np.random.default_rng(SEED + 100 + r)
    N = 1000
    lens = rng.integers(0, 4, M)
    rowStart = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    rr = np.repeat(np.arange(M), lens)
    cc = rng.integers(0, N, len(rr)).astype(np.int64)
    (out, dR, da), (w_out, w_dR, w_da) = _run_kernels(L, torch, rowStart, rr, cc, M, N, r, r, r, 0, rng)
    assert np.array_equal(out, w_out) and np.array_equal(dR, w_dR) and np.array_equal(da, w_da)


# ---- Algorithm.gatv2_scores / gatv2_backward at p = 1 -----------------------------------------------------------
@pytest.mark.parametrize("name", ALGS)
def test_p1_algorithm_scores_and_backward_all_algorithms(world, name):
    logM, npr, r = 8, 7, 8
    N = 1 << logM
    S = D.SpmatLocal.load_er(logM, npr, SEED)
    alg = D.Algorithm(name, S, r, 1)
    d = alg.dims
    rng = np.random.default_rng(SEED + 3)
    Av = rng.integers(-3, 4, (d.localArows, r)).astype(np.float64)
    Bv = rng.integers(-3, 4, (d.localBrows, r)).astype(np.float64)
    a_np = rng.integers(-2, 3, r).astype(np.float64)
    rc = {mode: coords(alg, mode) for mode in ("A", "B")}
    A, B = alg.like_A_matrix(), alg.like_B_matrix()
    A.from_host(Av)
    B.from_host(Bv)
    a = _vec(r)
    a.from_host(a_np)
    grads = {}
    for mode in ("A", "B"):
        rows, cols = rc[mode]
        out = (alg.like_S_values if mode == "A" else alg.like_ST_values)(float("nan"))
        alg.gatv2_scores(A, B, a, out, mode, EXACT_ALPHA)
        assert np.array_equal(out.to_host(), g2.scores_np(Av, Bv, rows, cols, a_np, EXACT_ALPHA)), (name, mode)
        gv = (alg.like_S_values if mode == "A" else alg.like_ST_values)(0.0)
        gv.from_host(((rows * 7 + cols * 3) % 5 - 2).astype(np.float64))  # the same function of (u, v) in both orders
        grads[mode] = gv
    dA, dB = alg.like_A_matrix(1.0), alg.like_B_matrix(-1.0)
    da = _vec(1, 5.0)
    for rep in range(2):
        dA.fill(1.0)
        dB.fill(-1.0)
        alg.gatv2_backward(A, B, a, grads["A"], grads["B"], dA, dB, da, EXACT_ALPHA)
        got = (dA.to_host(), dB.to_host(), da.to_host())
        if rep:
            assert all(np.array_equal(x, y) for x, y in zip(got, first)), name
        first = got
    rows, cols = rc["A"]
    g_np = ((rows * 7 + cols * 3) % 5 - 2).astype(np.float64)
    dA_inc, want_da = g2.grad_np(Av, Bv, rows, cols, g_np, a_np, EXACT_ALPHA)
    dB_inc, _ = g2.grad_np(Bv, Av, cols, rows, g_np, a_np, EXACT_ALPHA)
    assert np.array_equal(first[0], 1.0 + dA_inc), name
    assert np.array_equal(first[1], -1.0 + dB_inc), name
    assert np.array_equal(first[2], want_da), name
    # dA and dB may be the same matrix
    both = alg.like_A_matrix(0.0)
    alg.gatv2_backward(A, A, a, grads["A"], grads["B"], both, both, da, EXACT_ALPHA)
    s_inc, _ = g2.grad_np(Av, Av, rows, cols, g_np, a_np, EXACT_ALPHA)
    t_inc, _ = g2.grad_np(Av, Av, cols, rows, g_np, a_np, EXACT_ALPHA)
    assert np.array_equal(both.to_host(), s_inc + t_inc), name
    # bad orders, shapes and widths are refused
    from distributed_sddmm_b200 import lib
    assert lib().hnhd_alg_gatv2_scores(alg.h, A.h, B.h, a.h, alg.like_S_values(0.0).h, 2, 0.2) == -1
    with pytest.raises(RuntimeError, match="code -1"):
        alg.gatv2_scores(A, B, a, _vec(3), "B")  # a value vector of the wrong length
    with pytest.raises(RuntimeError, match="code -1"):
        alg.gatv2_scores(A, B, _vec(r - 1), alg.like_S_values(0.0), "A")
    with pytest.raises(RuntimeError, match="code -1"):
        alg.gatv2_backward(A, B, a, _vec(1), grads["B"], dA, dB, da)


# ---- GATv2 GAT at p = 1 ---------------------------------------------------------------------------------------
def _p1_net(name, logM=8, npr=6, attention="gatv2"):
    N = 1 << logM
    rows, cols, _ = orc.er_tuples(logM, npr, SEED)
    layers, X0, weights = gat_inputs(N, LAYERS, SEED)
    a = g2.attention_inputs(layers, SEED)
    S = D.SpmatLocal.load_er(logM, npr, SEED)
    alg = D.Algorithm(name, S, layers[0][0], 1)
    net = D.GAT(alg, layers, ALPHA, attention=attention)
    for i, (_, fph, heads) in enumerate(layers):
        for h in range(heads):
            net.set_weight(i, h, weights[i][h])
            net.set_attention_vectors(i, h, a[i][h], np.full(fph, 9.0))  # a2 is not read
    net.set_input(X0)
    G = np.random.default_rng(SEED + 5).uniform(-1, 1, net.buffer_shape(len(layers)))
    return dict(N=N, rows=rows, cols=cols, layers=layers, X0=X0, weights=weights, a=a, S=S, alg=alg, net=net, G=G)


def _oracle_args(P, weights=None, a=None):
    return (P["rows"], P["cols"], P["N"], P["layers"], P["weights"] if weights is None else weights,
            P["a"] if a is None else a, ALPHA, P["X0"])


@pytest.mark.parametrize("name", ALGS)
def test_p1_gatv2_matches_autograd(world, name):
    P = _p1_net(name)
    net, layers = P["net"], P["layers"]
    net.forward()
    out = net.buffer(len(layers))
    want = g2.gatv2_forward_global(*_oracle_args(P))
    assert np.abs(want).max() > 0
    assert rel_err(out, want) < 1e-10, name
    net.backward(P["G"])
    dX0, dW, da = g2.gatv2_backward_global(*_oracle_args(P), P["G"])
    assert np.abs(dX0).max() > 0
    assert rel_err(net.input_grad(), dX0) < 1e-10, name
    grads = {}
    for i, (_, _, heads) in enumerate(layers):
        for h in range(heads):
            assert np.abs(dW[i][h]).max() > 0 and np.abs(da[i][h]).max() > 0, (i, h)
            assert rel_err(net.weight_grad(i, h), dW[i][h]) < 1e-10, (name, i, h)
            g1, g2_ = net.attention_grads(i, h)
            assert rel_err(g1, da[i][h]) < 1e-10, (name, i, h)
            assert not g2_.any(), (name, i, h)
            grads[i, h] = (net.weight_grad(i, h), g1)
    # a second forward + backward is bit-identical
    dX_first = net.input_grad()
    net.forward()
    assert np.array_equal(net.buffer(len(layers)), out)
    net.backward(P["G"])
    assert np.array_equal(net.input_grad(), dX_first)
    for (i, h), (w, g1) in grads.items():
        assert np.array_equal(net.weight_grad(i, h), w) and np.array_equal(net.attention_grads(i, h)[0], g1), (i, h)


@pytest.mark.parametrize("name", ALGS)
def test_p1_gatv2_sgd_steps_track_autograd(world, name):
    """Three steps of (W, a) -= lr * gradient driven from Python follow the same three steps of the autograd model."""
    P = _p1_net(name)
    net, layers = P["net"], P["layers"]
    _, dW0, da0 = g2.gatv2_backward_global(*_oracle_args(P), P["G"])
    lr = 0.01 / max(np.abs(g).max() for nested in (dW0, da0) for per in nested for g in per)
    mine = [[[v.copy() for v in per] for per in P[k]] for k in ("weights", "a")]
    ref = [[[v.copy() for v in per] for per in P[k]] for k in ("weights", "a")]
    for step in range(3):
        net.forward()
        net.backward(P["G"])
        _, dW, da = g2.gatv2_backward_global(*_oracle_args(P, *ref), P["G"])
        for i, (_, fph, heads) in enumerate(layers):
            for h in range(heads):
                for k, g in enumerate((net.weight_grad(i, h), net.attention_grads(i, h)[0])):
                    mine[k][i][h] = mine[k][i][h] - lr * g
                for k, g in enumerate((dW, da)):
                    ref[k][i][h] = ref[k][i][h] - lr * g[i][h]
                net.set_weight(i, h, mine[0][i][h])
                net.set_attention_vectors(i, h, mine[1][i][h], np.zeros(fph))
    for k, key in enumerate(("weights", "a")):
        for i, (_, _, heads) in enumerate(layers):
            for h in range(heads):
                assert rel_err(mine[k][i][h], ref[k][i][h]) < 1e-9, (name, key, i, h)
                assert np.abs(ref[k][i][h] - P[key][i][h]).max() > 1e-3 * np.abs(P[key][i][h]).max()  # they moved
    net.forward()
    assert rel_err(net.buffer(len(layers)), g2.gatv2_forward_global(*_oracle_args(P, *ref))) < 1e-9


def test_p1_attention_switch_zero_vectors_and_validation(world):
    """A fresh GAT (a = 0) gives the same output under "gatv2" as under "additive", bit for bit; switching kinds
    leaves "leaky", "softmax" and "additive" bit-identical to fresh objects of those kinds; "GATv2" is refused with a
    message naming every kind; new attention vectors make the activations stale."""
    from distributed_sddmm_b200 import lib
    P = _p1_net("15d_fusion2", logM=7, npr=5, attention="leaky")
    net, layers = P["net"], P["layers"]
    assert lib().hnhd_gat_set_attention(net.h, b"GATv2") == -1
    msg = lib().hnh_last_error_string()
    assert all(k in msg for k in (b'"leaky"', b'"softmax"', b'"additive"', b'"gatv2"')), msg

    def fresh(kind):
        g = D.GAT(P["alg"], layers, ALPHA, attention=kind)
        for i, (_, _, heads) in enumerate(layers):
            for h in range(heads):
                g.set_weight(i, h, P["weights"][i][h])
        g.set_input(P["X0"])
        g.forward()
        return g

    mean_v2, mean_add = fresh("gatv2"), fresh("additive")
    assert np.array_equal(mean_v2.buffer(len(layers)), mean_add.buffer(len(layers)))
    del mean_v2, mean_add

    outs = {}
    for kind in ("leaky", "softmax", "additive", "gatv2", "leaky", "softmax", "additive"):
        net.set_attention(kind)
        with pytest.raises(RuntimeError, match="no forward pass"):
            net.backward(P["G"])
        net.forward()
        net.backward(P["G"])
        got = (net.buffer(len(layers)), net.input_grad(), net.weight_grad(1, 2))
        if kind in outs:
            assert all(np.array_equal(x, y) for x, y in zip(got, outs[kind])), kind
        outs[kind] = got
    for kind in ("leaky", "softmax", "additive"):
        f = fresh(kind)
        # the switched object holds the GATv2 attention vectors as a1 (and 9s as a2): give the fresh one the same
        for i, (_, fph, heads) in enumerate(layers):
            for h in range(heads):
                f.set_attention_vectors(i, h, P["a"][i][h], np.full(fph, 9.0))
        f.forward()
        f.backward(P["G"])
        got = (f.buffer(len(layers)), f.input_grad(), f.weight_grad(1, 2))
        assert all(np.array_equal(x, y) for x, y in zip(got, outs[kind])), kind
        del f
    assert not np.allclose(outs["gatv2"][0], outs["additive"][0])
    net.set_attention("gatv2")
    net.forward()
    net.set_attention_vectors(0, 1, P["a"][0][1], np.zeros(layers[0][1]))
    with pytest.raises(RuntimeError, match="no forward pass"):
        net.backward(P["G"])


def test_gat_v2_benchmark_records(world):
    S = D.SpmatLocal.load_er(10, 8, SEED)
    for app in ("gat_v2", "gat_v2_train"):
        rec = D.benchmark_algorithm(S, "15d_fusion2", 64, 1, fused=True, app=app, trials=1, warmup=0)
        assert rec["num_trials"] == 1 and rec["elapsed"] > 0, (app, rec)
