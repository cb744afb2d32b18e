"""Additive graph attention on the GPU at p = 1: the new kernels against numpy, Algorithm.additive_scores / edge_sums
on every algorithm in both value orders (the column keys against the S-columns recovered by SDDMMs of index columns),
and the additive GAT forward + backward (dX0, every dW, da1, da2) and three SGD steps against the autograd model of
tests/gat_additive_oracle.py.  Multi-rank cases live in tests/test_gat_additive_multirank_gpu.py."""
import ctypes as C

import numpy as np
import pytest

from distributed_sddmm_b200 import driver as D
from oracle import hnh_oracle as orc
from tests import gat_additive_oracle as gao
from tests.mp_edge_softmax_worker import coords
from tests.mp_worker import gat_inputs

pytestmark = pytest.mark.gpu
SEED = 0xC0FFEE + 4
ALGS = ["15d_fusion1", "15d_fusion2", "15d_sparse", "25d_dense_replicate", "25d_sparse_replicate"]
LAYERS = [[12, 8, 2], [16, 4, 3]]
ALPHA = 0.2


def rel_err(got, ref):
    return np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-300)


def leaky(x, alpha=ALPHA):
    return np.maximum(x, 0.0) + np.minimum(x, 0.0) * alpha


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
def test_node_scalars_and_rank2_update_against_numpy(world):
    import torch
    from distributed_sddmm_b200 import lib
    L = lib()
    dev = torch.device("cuda:0")
    st = torch.cuda.current_stream().cuda_stream
    rng = np.random.default_rng(41)
    f64 = dict(dtype=torch.float64, device=dev)
    # d even and 16-byte aligned (paired loads), d odd, and d even at an 8-byte offset (scalar loads)
    for n, d, shift in ((3000, 256, 0), (517, 7, 0), (300, 12, 1), (5, 1, 0)):
        P_np = rng.uniform(-1, 1, (n, d))
        a1_np, a2_np = rng.uniform(-1, 1, d), rng.uniform(-1, 1, d)
        P = torch.zeros(n * d + shift, **f64)
        P[shift:] = torch.from_numpy(P_np.ravel())
        a = torch.zeros(2 * d + 2 * shift, **f64)
        a[shift:shift + d] = torch.from_numpy(a1_np)
        a[d + 2 * shift:] = torch.from_numpy(a2_np)
        a1p, a2p = a.data_ptr() + 8 * shift, a.data_ptr() + 8 * (d + 2 * shift)
        s, t = torch.full((n,), float("nan"), **f64), torch.full((n,), float("nan"), **f64)
        D.check(L.hnh_gat_node_scalars_f64(s.data_ptr(), t.data_ptr(), P.data_ptr() + 8 * shift, a1p, a2p, n, d, st))
        torch.cuda.synchronize()
        assert rel_err(s.cpu().numpy(), P_np @ a1_np) < 1e-13, (n, d, shift)
        assert rel_err(t.cpu().numpy(), P_np @ a2_np) < 1e-13, (n, d, shift)
        s2, t2 = torch.empty_like(s), torch.empty_like(t)
        D.check(L.hnh_gat_node_scalars_f64(s2.data_ptr(), t2.data_ptr(), P.data_ptr() + 8 * shift, a1p, a2p, n, d, st))
        torch.cuda.synchronize()
        assert torch.equal(s, s2) and torch.equal(t, t2)
        # rank-2 row update on the same P
        ds_np, dt_np = rng.uniform(-1, 1, n), rng.uniform(-1, 1, n)
        ds, dt = torch.from_numpy(ds_np).to(dev), torch.from_numpy(dt_np).to(dev)
        D.check(L.hnh_gat_rank2_update_f64(P.data_ptr() + 8 * shift, ds.data_ptr(), dt.data_ptr(), a1p, a2p, n, d, st))
        torch.cuda.synchronize()
        want = P_np + np.outer(ds_np, a1_np) + np.outer(dt_np, a2_np)
        assert rel_err(P[shift:].cpu().numpy().reshape(n, d), want) < 1e-14, (n, d, shift)


def test_edge_scores_and_sums_against_numpy(world):
    import torch
    from distributed_sddmm_b200 import lib
    L = lib()
    dev = torch.device("cuda:0")
    st = torch.cuda.current_stream().cuda_stream
    rng = np.random.default_rng(43)
    nr, nc, n = 700, 650, 40000
    rk, ck = rng.integers(0, nr, n), rng.integers(0, nc, n)
    rk[:5000] = 5  # a row of several plan pieces
    ck[5000:7000] = nc - 1
    s_np, t_np = rng.uniform(-1, 1, nr), rng.uniform(-1, 1, nc)
    s_np[0] = -t_np[0]  # s + t == 0 exactly on some entries: LeakyReLU'(0) = alpha
    rk[::9], ck[::9] = 0, 0
    I32 = dict(dtype=torch.int32, device=dev)
    rkd, ckd = torch.from_numpy(rk.astype(np.int32)).to(dev), torch.from_numpy(ck.astype(np.int32)).to(dev)
    s, t = torch.from_numpy(s_np).to(dev), torch.from_numpy(t_np).to(dev)
    x = s_np[rk] + t_np[ck]
    assert (x > 0).any() and (x < 0).any() and (x == 0).any()
    for derivative, want in ((0, leaky(x)), (1, np.where(x > 0, 1.0, ALPHA))):
        out = torch.full((n,), float("nan"), dtype=torch.float64, device=dev)
        D.check(L.hnh_gat_edge_scores_f64(out.data_ptr(), s.data_ptr(), t.data_ptr(), rkd.data_ptr(), ckd.data_ptr(), n, ALPHA,
                                          derivative, st))
        torch.cuda.synchronize()
        assert np.array_equal(out.cpu().numpy(), want), derivative
    # row and column sums over a plan keyed by row / column
    v_np = rng.uniform(-1, 1, n)
    v = torch.from_numpy(v_np).to(dev)
    for keys, keys_d, K in ((rk, rkd, nr), (ck, ckd, nc)):
        cap = L.hnh_edge_softmax_piece_bound(n, K)
        perm, rs, pf = torch.empty(n, **I32), torch.empty(K + 1, **I32), torch.empty(K + 1, **I32)
        pr = torch.empty(max(cap, 1), **I32)
        npieces = C.c_int64(-1)
        D.check(L.hnh_edge_softmax_plan(keys_d.data_ptr(), n, K, perm.data_ptr(), rs.data_ptr(), pf.data_ptr(), pr.data_ptr(), cap,
                                        C.byref(npieces), st))
        sums = []
        for _ in range(2):
            ps = torch.full((max(npieces.value, 1),), float("nan"), dtype=torch.float64, device=dev)
            out = torch.full((K,), float("nan"), dtype=torch.float64, device=dev)
            D.check(L.hnh_edge_sum_f64(v.data_ptr(), perm.data_ptr(), rs.data_ptr(), pf.data_ptr(), pr.data_ptr(), K, npieces.value,
                                       ps.data_ptr(), out.data_ptr(), st))
            torch.cuda.synchronize()
            sums.append(out.cpu().numpy())
        want = np.bincount(keys, weights=v_np, minlength=K)
        assert np.abs(sums[0] - want).max() < 1e-12 * np.abs(v_np).sum()
        assert np.all(sums[0][np.bincount(keys, minlength=K) == 0] == 0)
        assert np.array_equal(sums[0], sums[1])  # bit-identical repeat


# ---- Algorithm.additive_scores / edge_sums at p = 1 -------------------------------------------------------------
@pytest.mark.parametrize("name", ALGS)
def test_p1_column_keys_scores_and_sums_all_algorithms(world, name):
    logM, npr, R = 8, 7, 8
    N = 1 << logM
    S = D.SpmatLocal.load_er(logM, npr, SEED)
    alg = D.Algorithm(name, S, R, 1)
    zero, index = _vec(N), _vec(N)
    index.from_host(np.arange(N, dtype=np.float64))
    for mode in ("A", "B"):
        r, c = coords(alg, mode)
        like = alg.like_S_values if mode == "A" else alg.like_ST_values
        out = like(-1.0)
        # s = node index, t = 0 gives each entry's row key; s = 0, t = node index its column key
        alg.additive_scores(index, zero, out, mode)
        assert np.array_equal(out.to_host(), r), (name, mode)
        alg.additive_scores(zero, index, out, mode)
        assert np.array_equal(out.to_host(), c), (name, mode)
        # scores of random node scalars, and their derivative
        rng = np.random.default_rng(7)
        s_np, t_np = rng.uniform(-1, 1, N), rng.uniform(-1, 1, N)
        s, t = _vec(N), _vec(N)
        s.from_host(s_np)
        t.from_host(t_np)
        alg.additive_scores(s, t, out, mode, ALPHA)
        assert np.array_equal(out.to_host(), leaky(s_np[r] + t_np[c])), (name, mode)
        alg.additive_scores(s, t, out, mode, ALPHA, derivative=True)
        assert np.array_equal(out.to_host(), np.where(s_np[r] + t_np[c] > 0, 1.0, ALPHA)), (name, mode)
    # row and column sums of an A-order vector
    r, c = coords(alg, "A")
    v_np = np.cos(0.3 * r + 0.7 * c)
    v = alg.like_S_values(0.0)
    v.from_host(v_np)
    rows, cols = _vec(N + 3, 5.0), _vec(N, 5.0)
    alg.edge_sums(v, rows, cols)
    got_r, got_c = rows.to_host(), cols.to_host()
    assert rel_err(got_r[:N], np.bincount(r, weights=v_np, minlength=N)) < 1e-13, name
    assert np.all(got_r[N:] == 0)
    assert rel_err(got_c, np.bincount(c, weights=v_np, minlength=N)) < 1e-13, name
    alg.edge_sums(v, rows, cols)
    assert np.array_equal(rows.to_host(), got_r) and np.array_equal(cols.to_host(), got_c)
    # short node vectors are refused
    with pytest.raises(RuntimeError, match="code -1"):
        alg.additive_scores(_vec(N - 1), zero, alg.like_S_values(0.0), "A")
    with pytest.raises(RuntimeError, match="code -1"):
        alg.edge_sums(v, _vec(N), _vec(N - 1))


# ---- additive graph attention at p = 1 ------------------------------------------------------------------------
def _p1_net(name, logM=8, npr=6, attention="additive"):
    N = 1 << logM
    rows, cols, _ = orc.er_tuples(logM, npr, SEED)
    layers, X0, weights = gat_inputs(N, LAYERS, SEED)
    a1, a2 = gao.attention_inputs(layers, SEED)
    S = D.SpmatLocal.load_er(logM, npr, SEED)
    alg = D.Algorithm(name, S, layers[0][0], 1)
    net = D.GAT(alg, layers, ALPHA, attention=attention)
    for i, (_, _, heads) in enumerate(layers):
        for h in range(heads):
            net.set_weight(i, h, weights[i][h])
            net.set_attention_vectors(i, h, a1[i][h], a2[i][h])
    net.set_input(X0)
    G = np.random.default_rng(SEED + 5).uniform(-1, 1, net.buffer_shape(len(layers)))
    return dict(N=N, rows=rows, cols=cols, layers=layers, X0=X0, weights=weights, a1=a1, a2=a2, S=S, alg=alg, net=net, G=G)


def _oracle_args(P, weights=None, a1=None, a2=None):
    return (P["rows"], P["cols"], P["N"], P["layers"], P["weights"] if weights is None else weights,
            P["a1"] if a1 is None else a1, P["a2"] if a2 is None else a2, ALPHA, P["X0"])


@pytest.mark.parametrize("name", ALGS)
def test_p1_additive_gat_matches_autograd(world, name):
    P = _p1_net(name)
    net, layers = P["net"], P["layers"]
    net.forward()
    out = net.buffer(len(layers))
    want = gao.gat_additive_forward_global(*_oracle_args(P))
    assert np.abs(want).max() > 0
    assert rel_err(out, want) < 1e-10, name
    net.backward(P["G"])
    dX0, dW, da1, da2 = gao.gat_additive_backward_global(*_oracle_args(P), P["G"])
    assert np.abs(dX0).max() > 0
    assert rel_err(net.input_grad(), dX0) < 1e-10, name
    grads = {}
    for i, (_, _, heads) in enumerate(layers):
        for h in range(heads):
            assert np.abs(dW[i][h]).max() > 0 and np.abs(da1[i][h]).max() > 0 and np.abs(da2[i][h]).max() > 0, (i, h)
            assert rel_err(net.weight_grad(i, h), dW[i][h]) < 1e-10, (name, i, h)
            g1, g2 = net.attention_grads(i, h)
            assert rel_err(g1, da1[i][h]) < 1e-10, (name, i, h)
            assert rel_err(g2, da2[i][h]) < 1e-10, (name, i, h)
            grads[i, h] = (net.weight_grad(i, h), g1, g2)
    # the backward pass leaves the activations alone; a second forward + backward is bit-identical
    assert np.array_equal(net.buffer(len(layers)), out)
    dX_first = net.input_grad()
    net.forward()
    assert np.array_equal(net.buffer(len(layers)), out)
    net.backward(P["G"])
    assert np.array_equal(net.input_grad(), dX_first)
    for (i, h), (w, g1, g2) in grads.items():
        n1, n2 = net.attention_grads(i, h)
        assert np.array_equal(net.weight_grad(i, h), w) and np.array_equal(n1, g1) and np.array_equal(n2, g2), (i, h)


@pytest.mark.parametrize("name", ALGS)
def test_p1_additive_gat_sgd_steps_track_autograd(world, name):
    """Three steps of (W, a1, a2) -= lr * gradient driven from Python follow the same three steps of the autograd
    model."""
    P = _p1_net(name)
    net, layers = P["net"], P["layers"]
    _, dW0, da10, da20 = gao.gat_additive_backward_global(*_oracle_args(P), P["G"])
    lr = 0.01 / max(np.abs(g).max() for nested in (dW0, da10, da20) for per in nested for g in per)
    mine = [[[v.copy() for v in per] for per in P[k]] for k in ("weights", "a1", "a2")]
    ref = [[[v.copy() for v in per] for per in P[k]] for k in ("weights", "a1", "a2")]
    for step in range(3):
        net.forward()
        net.backward(P["G"])
        _, dW, da1, da2 = gao.gat_additive_backward_global(*_oracle_args(P, *ref), P["G"])
        for i, (_, _, heads) in enumerate(layers):
            for h in range(heads):
                g1, g2 = net.attention_grads(i, h)
                for k, g in enumerate((net.weight_grad(i, h), g1, g2)):
                    mine[k][i][h] = mine[k][i][h] - lr * g
                for k, g in enumerate((dW, da1, da2)):
                    ref[k][i][h] = ref[k][i][h] - lr * g[i][h]
                net.set_weight(i, h, mine[0][i][h])
                net.set_attention_vectors(i, h, mine[1][i][h], mine[2][i][h])
    for k, key in enumerate(("weights", "a1", "a2")):
        for i, (_, _, heads) in enumerate(layers):
            for h in range(heads):
                assert rel_err(mine[k][i][h], ref[k][i][h]) < 1e-9, (name, key, i, h)
                assert np.abs(ref[k][i][h] - P[key][i][h]).max() > 1e-3 * np.abs(P[key][i][h]).max()  # they moved
    net.forward()
    want = gao.gat_additive_forward_global(*_oracle_args(P, *ref))
    assert rel_err(net.buffer(len(layers)), want) < 1e-9


def test_p1_attention_switch_and_validation(world):
    """Switching between "leaky", "softmax" and "additive" leaves the first two bit-identical to a fresh object of
    that kind; the attention vectors make the activations stale; the new C entry points validate layer, head, kind
    and that a backward pass has run."""
    from distributed_sddmm_b200 import lib
    L = lib()
    P = _p1_net("15d_fusion2", logM=7, npr=5, attention="leaky")
    net, layers = P["net"], P["layers"]
    fph = layers[0][1]
    buf = (C.c_double * fph)()
    p = C.addressof(buf)
    # nothing computed yet
    assert L.hnhd_gat_get_attention_grads(net.h, 0, 0, p, p) == -1
    assert b"no backward pass" in L.hnh_last_error_string()
    # bad layer / head / pointer / kind
    assert L.hnhd_gat_set_attention_vectors(net.h, len(layers), 0, p, p) == -1
    assert b"no such layer" in L.hnh_last_error_string()
    assert L.hnhd_gat_set_attention_vectors(net.h, -1, 0, p, p) == -1
    assert L.hnhd_gat_set_attention_vectors(net.h, 0, layers[0][2], p, p) == -1
    assert b"no such head" in L.hnh_last_error_string()
    assert L.hnhd_gat_set_attention_vectors(net.h, 0, 0, p, None) == -1
    assert L.hnhd_gat_get_attention_grads(net.h, 1, -1, p, p) == -1
    assert b"no such head" in L.hnh_last_error_string()
    assert L.hnhd_gat_get_attention_grads(net.h, 2, 0, p, p) == -1
    assert L.hnhd_gat_set_attention(net.h, b"Additive") == -1
    assert b"additive" in L.hnh_last_error_string()

    outs = {}
    for kind in ("leaky", "softmax", "additive", "leaky", "softmax"):
        net.set_attention(kind)
        with pytest.raises(RuntimeError, match="no forward pass"):
            net.backward(P["G"])
        net.forward()
        net.backward(P["G"])
        got = (net.buffer(len(layers)), net.input_grad(), net.weight_grad(1, 2))
        if kind in outs:
            assert all(np.array_equal(a, b) for a, b in zip(got, outs[kind])), kind
        outs[kind] = got
        if kind != "additive":  # a1 / a2 do not enter: their gradients are zero
            assert all(not g.any() for g in net.attention_grads(1, 1)), kind
    for kind in ("leaky", "softmax"):
        fresh = D.GAT(P["alg"], layers, ALPHA, attention=kind)
        for i, (_, _, heads) in enumerate(layers):
            for h in range(heads):
                fresh.set_weight(i, h, P["weights"][i][h])
        fresh.set_input(P["X0"])
        fresh.forward()
        fresh.backward(P["G"])
        got = (fresh.buffer(len(layers)), fresh.input_grad(), fresh.weight_grad(1, 2))
        assert all(np.array_equal(a, b) for a, b in zip(got, outs[kind])), kind
        del fresh
    assert not np.allclose(outs["additive"][0], outs["softmax"][0])
    # new attention vectors make the activations stale
    net.set_attention("additive")
    net.forward()
    net.set_attention_vectors(0, 1, P["a1"][0][1], P["a2"][0][1])
    with pytest.raises(RuntimeError, match="no forward pass"):
        net.backward(P["G"])


def test_p1_zero_attention_vectors_give_mean_aggregation(world):
    """A fresh GAT's a1 / a2 are zero: additive attention is then the mean over each node's neighbours."""
    P = _p1_net("15d_fusion1", logM=7, npr=5)
    fresh = D.GAT(P["alg"], P["layers"], ALPHA, attention="additive")
    for i, (_, _, heads) in enumerate(P["layers"]):
        for h in range(heads):
            fresh.set_weight(i, h, P["weights"][i][h])
    fresh.set_input(P["X0"])
    fresh.forward()
    zeros = [[np.zeros(fph) for _ in range(heads)] for _, fph, heads in P["layers"]]
    want = gao.gat_additive_forward_global(*_oracle_args(P, None, zeros, zeros))
    assert rel_err(fresh.buffer(len(P["layers"])), want) < 1e-10


def test_gat_additive_benchmark_records(world):
    S = D.SpmatLocal.load_er(10, 8, SEED)
    for app in ("gat_additive", "gat_additive_train"):
        rec = D.benchmark_algorithm(S, "15d_fusion1", R=32, c=1, fused=True, app=app, trials=1, warmup=0)
        assert rec["overall_throughput"] > 0 and rec["elapsed"] > 0, app
