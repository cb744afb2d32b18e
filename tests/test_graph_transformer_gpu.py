"""Graph transformer on the GPU on one rank: forward output, input gradient and every parameter gradient against the
fp64 model of tests/graph_transformer_oracle.py to a relative error of 1e-10, for 1-3 layers, every (gate, edge)
combination and attention dropout 0 and 0.3; head widths 32, 64 and 256 and an odd width that takes the generic
attention kernels and the scalar gate path; duplicate entries and empty rows; the gate kernels past one resident wave
and on misaligned rows; repeats bit-identical; the refusal to run a backward pass on stale activations.  Multi-rank
cases live in tests/test_graph_transformer_multirank_gpu.py."""
import numpy as np
import pytest

from distributed_sddmm_b200 import driver as D
from oracle import hnh_oracle as orc
from tests import graph_transformer_oracle as gto
from tests.test_sparse_attention_bias import _pattern

pytestmark = pytest.mark.gpu
SEED = 0xC0FFEE + 71


def rel_err(got, ref):
    return np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-300)


def grad_err(got, ref, scale):
    """Relative error against the larger of ref's largest entry and `scale` (the layer's largest gradient entry): the
    key bias gradient is 0 up to rounding (a key bias shifts every score of a row alike)."""
    return np.abs(got - ref).max() / max(np.abs(ref).max(), scale, 1e-300)


def attr_of(rows, cols, e):
    """Edge attributes as a function of the global S-row and S-column only."""
    rows, cols = np.asarray(rows, np.float64), np.asarray(cols, np.float64)
    return np.cos(0.31 * rows[:, None] + 0.73 * cols[:, None] + 0.45 * np.arange(e)[None, :])


@pytest.fixture(scope="module")
def world():
    D.world_init("self")
    yield
    D.world_finalize()


def build(layers, edge_dim, beta, logM=7, npr=5, alg_name="15d_fusion1", pattern=None, seed=SEED):
    """The network on one rank with random parameters, input and edge attributes; returns a dict of everything."""
    N = 1 << logM
    if pattern is None:
        rows, cols, _ = orc.er_tuples(logM, npr, seed)
    else:
        rows, cols = pattern
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    S = D.SpmatLocal.from_tuples(N, N, rows, cols, np.ones(len(rows)))
    alg = D.Algorithm(alg_name, S, layers[0][0], 1)
    net = D.GraphTransformer(alg, layers, edge_dim=edge_dim, beta=beta)
    rng = np.random.default_rng(seed + 1)
    params = gto.random_params(layers, edge_dim, beta, rng)
    for l, P in enumerate(params):
        for name, v in P.items():
            net.set_param(l, name, v)
    X = rng.uniform(-1, 1, (N, layers[0][0]))
    Xl = np.zeros(net.buffer_shape(0))
    Xl[:N] = X
    net.set_input(Xl)
    if edge_dim:
        net.set_edge_attributes(attr_of(*alg.entry_coordinates("A"), edge_dim), attr_of(*alg.entry_coordinates("B"), edge_dim))
    shape = net.buffer_shape(len(layers))
    G = np.zeros(shape)
    G[:N] = rng.uniform(-1, 1, (N, shape[1]))
    return dict(N=N, rows=rows, cols=cols, S=S, alg=alg, net=net, params=params, X=X, G=G, layers=layers,
                attr=attr_of(rows, cols, edge_dim) if edge_dim else None, beta=beta)


def check_against_model(P, dropout, seed):
    net, N, layers = P["net"], P["N"], P["layers"]
    net.forward(dropout, seed)
    args = (P["rows"], P["cols"], N, layers, P["params"], P["X"])
    kw = dict(attr=P["attr"], beta=P["beta"], p=dropout, seed=seed)
    want = gto.forward_np(*args, **kw)
    out = net.buffer(len(layers))[:N]
    assert np.abs(want).max() > 0
    assert rel_err(out, want) < 1e-10
    net.backward(P["G"])
    dX, dP = gto.backward_np(*args, P["G"][:N], **kw)
    assert rel_err(net.input_grad()[:N], dX) < 1e-10
    for l, grads in enumerate(dP):
        scale = max(np.abs(g).max() for g in grads.values())
        for name, g in grads.items():
            got = net.param_grad(l, name)
            assert got.shape == g.shape, (l, name)
            assert grad_err(got, g, scale) < 1e-10, (l, name, grad_err(got, g, scale))


LAYER_SETS = {1: [(6, 4, 2)], 2: [(6, 4, 2), (8, 3, 3)], 3: [(6, 4, 2), (8, 3, 3), (9, 8, 1)]}


@pytest.mark.parametrize("dropout", [0.0, 0.3])
@pytest.mark.parametrize("beta", [False, True])
@pytest.mark.parametrize("edge_dim", [0, 3])
@pytest.mark.parametrize("n_layers", [1, 2, 3])
def test_matches_model(world, n_layers, edge_dim, beta, dropout):
    P = build(LAYER_SETS[n_layers], edge_dim, beta)
    check_against_model(P, dropout, 17)


@pytest.mark.parametrize("d", [32, 64, 256, 5])
def test_head_widths(world, d):
    """Widths of the attention kernels' table and an odd one (r = 15: the generic attention kernels and the scalar gate
    path)."""
    H = 3 if d == 5 else 2 if d < 256 else 1
    P = build([(7, d, H), (d * H, 4, 2)], 2, True, logM=6)
    check_against_model(P, 0.3, 5)


@pytest.mark.parametrize("alg_name", ["15d_fusion2", "15d_sparse", "25d_dense_replicate", "25d_sparse_replicate"])
def test_duplicates_and_empty_rows(world, alg_name):
    """A pattern with duplicate entries and empty rows, on every algorithm at p = 1."""
    rng = np.random.default_rng(9)
    rows, cols = _pattern(rng, 64, 64, per_row=6)
    rows, cols = np.concatenate([rows, [5, 5, 5]]), np.concatenate([cols, [9, 9, 9]])
    P = build(LAYER_SETS[2], 3, True, logM=6, alg_name=alg_name, pattern=(rows, cols))
    check_against_model(P, 0.3, 23)


def test_backward_repeats_bit_identical(world):
    P = build(LAYER_SETS[3], 3, True)
    net, layers = P["net"], P["layers"]
    net.forward(0.3, 99)
    out = net.buffer(len(layers))
    net.backward(P["G"])
    first = [net.input_grad()] + [net.param_grad(l, n) for l in range(len(layers)) for n in net.param_names()]
    net.backward(P["G"])
    second = [net.input_grad()] + [net.param_grad(l, n) for l in range(len(layers)) for n in net.param_names()]
    assert all(np.array_equal(a, b) for a, b in zip(first, second))
    net.forward(0.3, 99)
    assert np.array_equal(net.buffer(len(layers)), out)


def test_backward_needs_a_current_forward_pass(world):
    P = build(LAYER_SETS[2], 3, False, logM=6)
    net = P["net"]
    with pytest.raises(RuntimeError, match="code -1.*no forward pass"):
        net.backward(P["G"])
    with pytest.raises(RuntimeError, match="code -1.*no backward pass"):
        net.param_grad(0, "query")
    with pytest.raises(RuntimeError, match="code -1.*no backward pass"):
        net.input_grad()
    net.forward()
    net.backward(P["G"])
    for change in (lambda: net.set_param(1, "skip_bias", P["params"][1]["skip_bias"]),
                   lambda: net.set_input(np.zeros(net.buffer_shape(0))),
                   lambda: net.set_edge_attributes(attr_of(*P["alg"].entry_coordinates("A"), 3),
                                                   attr_of(*P["alg"].entry_coordinates("B"), 3))):
        change()
        with pytest.raises(RuntimeError, match="no forward pass"):
            net.backward(P["G"])
        net.forward()
        net.backward(P["G"])
    with pytest.raises(ValueError):
        net.backward(P["G"][:, :-1])


def test_model_arguments_are_refused(world):
    """Bad layer chains, unknown parameters, wrong attribute counts and a missing edge attribute are refused with
    HNH_E_INVALID before any launch."""
    N = 64
    rows, cols, _ = orc.er_tuples(6, 4, SEED)
    S = D.SpmatLocal.from_tuples(N, N, rows, cols, np.ones(len(rows)))
    alg = D.Algorithm("15d_fusion1", S, 6, 1)
    for layers in ([(6, 4, 2), (7, 3, 3)], [(6, 0, 2)], [(6, 4, -1)]):
        with pytest.raises(RuntimeError, match="code -1"):
            D.GraphTransformer(alg, layers)
    import ctypes as C
    from distributed_sddmm_b200 import lib
    h = C.c_void_p()
    assert lib().hnhd_gt_create(alg.h, 1, (C.c_int * 3)(6, 4, 2), -1, 0, C.byref(h)) == -1
    assert b"edge_dim" in lib().hnh_last_error_string()
    net = D.GraphTransformer(alg, [(6, 4, 2)])
    for name in ("edge", "beta", "nope"):
        with pytest.raises(RuntimeError, match="code -1.*no parameter"):
            net.param_shape(0, name)
    with pytest.raises(RuntimeError, match="code -1.*no such layer"):
        net.param_shape(1, "query")
    assert net.param_shape(0, "query") == (6, 8) and net.param_shape(0, "key_bias") == (8,)
    with pytest.raises(ValueError):
        net.set_param(0, "query", np.zeros((8, 6)))
    assert lib().hnhd_gt_forward(net.h, 1.0, 0) == -1 and b"dropout" in lib().hnh_last_error_string()
    edged = D.GraphTransformer(alg, [(6, 4, 2)], edge_dim=2, beta=True)
    assert edged.param_shape(0, "edge") == (2, 8) and edged.param_shape(0, "beta") == (24,)
    with pytest.raises(RuntimeError, match="code -1.*no edge attributes"):
        edged.forward()
    nA, nB = len(alg.like_S_values()), len(alg.like_ST_values())
    with pytest.raises(RuntimeError, match="code -1.*entries"):
        edged.set_edge_attributes(np.zeros((nA + 1, 2)), np.zeros((nB, 2)))
    with pytest.raises(RuntimeError, match="code -1.*entries"):
        edged.set_edge_attributes(np.zeros((nA, 2)), np.zeros((nB - 1, 2)))
    edged.set_edge_attributes(np.zeros((nA, 2)), np.zeros((nB, 2)))
    edged.forward()


@pytest.mark.parametrize("r", [6, 7])
def test_gate_kernels_past_one_wave(world, r):
    """n = 50000 rows (more than a resident wave of the row kernels), an even and an odd width, and rows shifted by
    one double (misaligned: the scalar path); the gate forward with and without ReLU and gate vector, its backward,
    and the bias add, against numpy; dw_beta bit-identical over repeats."""
    import torch
    from distributed_sddmm_b200 import check, lib
    L = lib()
    st = torch.cuda.current_stream().cuda_stream
    rng = np.random.default_rng(r)
    n = 50000
    M, R, G = (rng.uniform(-1, 1, (n, r)) for _ in range(3))
    w = rng.uniform(-1, 1, 3 * r)
    b = rng.uniform(-1, 1, r)
    for shift in (0, 1):
        def dev(x):
            t = torch.zeros(x.size + 1, dtype=torch.float64, device="cuda")
            t[shift:shift + x.size] = torch.from_numpy(x.reshape(-1))
            return t
        def ptr(t):
            return t.data_ptr() + 8 * shift
        def host(t, shape):
            torch.cuda.synchronize()
            return t[shift:shift + int(np.prod(shape))].cpu().numpy().reshape(shape)
        dM_, dR_, dX = dev(M), dev(R), dev(M)
        check(L.hnh_row_bias_add_f64(ptr(dX), ptr(dev(b)), n, r, st), "row_bias_add")
        assert np.array_equal(host(dX, (n, r)), M + b)
        for gate in (False, True):
            beta = 1 / (1 + np.exp(-(np.concatenate([M, R, M - R], 1) @ w)))[:, None] if gate else None
            Yraw = beta * R + (1 - beta) * M if gate else M + R
            dw_d = dev(w)
            for relu in (0, 1):
                Y = dev(np.full((n, r), np.nan))
                check(L.hnh_gt_gate_f64(ptr(Y), ptr(dM_), ptr(dR_), ptr(dw_d) if gate else None, n, r, relu, st), "gate")
                Yw = np.maximum(Yraw, 0) if relu else Yraw
                Yh = host(Y, (n, r))
                assert rel_err(Yh, Yw) < 1e-13, (shift, gate, relu)
                dY = np.where(Yh > 0, G, 0.0) if relu else G
                ws_bytes = L.hnh_gt_gate_backward_workspace_bytes(n, r)
                ws = torch.full((ws_bytes // 8,), np.nan, dtype=torch.float64, device="cuda")
                outs = [dev(np.full((n, r), np.nan)) for _ in range(2)] + [dev(np.full(3 * r, np.nan))]
                dws = []
                for _ in range(2):
                    check(L.hnh_gt_gate_backward_f64(ptr(outs[0]), ptr(outs[1]), ptr(outs[2]) if gate else None, ptr(dev(G)),
                                                     ptr(Y) if relu else None, ptr(dM_), ptr(dR_), ptr(dw_d) if gate else None,
                                                     n, r, relu, ws.data_ptr(), ws_bytes, st), "gate_backward")
                    dws.append(host(outs[2], (3 * r,)).copy())
                if gate:
                    ds = (dY * (R - M)).sum(1, keepdims=True) * beta * (1 - beta)
                    w1, w2, w3 = w[:r], w[r:2 * r], w[2 * r:]
                    assert rel_err(host(outs[0], (n, r)), (1 - beta) * dY + ds * (w1 + w3)) < 1e-12
                    assert rel_err(host(outs[1], (n, r)), beta * dY + ds * (w2 - w3)) < 1e-12
                    assert rel_err(dws[0], (ds * np.concatenate([M, R, M - R], 1)).sum(0)) < 1e-11
                    assert np.array_equal(dws[0], dws[1])
                else:
                    assert np.array_equal(host(outs[0], (n, r)), dY) and np.array_equal(host(outs[1], (n, r)), dY)


def test_graph_transformer_benchmark_records(world):
    S = D.SpmatLocal.load_er(10, 8, SEED)
    for app in ("graph_transformer", "graph_transformer_train"):
        rec = D.benchmark_algorithm(S, "15d_fusion1", R=256, c=1, fused=True, app=app, trials=1, warmup=0)
        assert rec["overall_throughput"] > 0 and rec["elapsed"] > 0
