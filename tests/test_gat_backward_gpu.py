"""GAT backward pass on the GPU: the new device kernels against numpy, and forward + backward on one rank (every
algorithm has full-width operands there) against the autograd model of tests/gat_backward_oracle.py.
Multi-rank cases live in tests/test_gat_backward_multirank_gpu.py."""
import numpy as np
import pytest

from distributed_sddmm_b200 import driver as D
from oracle import hnh_oracle as orc
from tests import gat_backward_oracle as gbo
from tests.mp_worker import gat_inputs

pytestmark = pytest.mark.gpu
SEED = 0xC0FFEE + 3
ALGS = ["15d_fusion1", "15d_fusion2", "15d_sparse", "25d_dense_replicate", "25d_sparse_replicate"]
LAYERS = [[12, 8, 2], [16, 4, 3]]


def rel_err(got, ref):
    return np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-300)


@pytest.fixture(scope="module")
def world():
    D.world_init("self")
    yield
    D.world_finalize()


@pytest.fixture(scope="module")
def dev():
    import torch
    return torch.device("cuda:0")


def _tn(L, torch, dev, A, B):
    """C = A^T B through hnh_dgemm_tn_f64 (A, B torch tensors on the device); C NaN-prefilled."""
    from distributed_sddmm_b200 import lib  # noqa: F401
    k, m = A.shape
    n = B.shape[1]
    st = torch.cuda.current_stream().cuda_stream
    ws_bytes = L.hnh_dgemm_tn_workspace_bytes(m, n, k)
    assert ws_bytes >= 0
    ws = torch.full((max(ws_bytes, 8) // 8,), float("nan"), dtype=torch.float64, device=dev)
    C = torch.full((m, n), float("nan"), dtype=torch.float64, device=dev)
    D.check(L.hnh_dgemm_tn_f64(C.data_ptr(), A.data_ptr(), B.data_ptr(), m, n, k, ws.data_ptr(), ws_bytes, st))
    torch.cuda.synchronize()
    return C


def test_dgemm_tn_against_numpy(world, dev):
    """C (m x n) = A^T B for ragged shapes: one K step and many, one split of k and many, more output tiles than a
    wave of CTAs; NaN-prefilled output and workspace; two calls bit-identical."""
    import torch
    from distributed_sddmm_b200 import lib
    L = lib()
    rng = np.random.default_rng(21)
    for m, n, k in ((70, 11, 19), (1, 1, 1), (64, 64, 16), (300, 130, 5000), (130, 70, 100000), (1500, 1100, 700),
                    (5, 200, 3)):
        A, B = rng.uniform(-1, 1, (k, m)), rng.uniform(-1, 1, (k, n))
        dA, dB = torch.from_numpy(A).to(dev), torch.from_numpy(B).to(dev)
        C1 = _tn(L, torch, dev, dA, dB)
        assert rel_err(C1.cpu().numpy(), A.T @ B) < 1e-13, (m, n, k)
        C2 = _tn(L, torch, dev, dA, dB)
        assert torch.equal(C1, C2), (m, n, k)


def test_dgemm_tn_benchmark_shape(world, dev):
    """k = 2^20 rows, m = 1024, n = 256 (the weight gradient of the benchmark's widest layer).  Small-integer operands
    make every partial sum exact in fp64, so the result must equal the exact product bit for bit whatever the order
    of summation; two calls are bit-identical."""
    import torch
    from distributed_sddmm_b200 import lib
    L = lib()
    k, m, n = 1 << 20, 1024, 256
    g = torch.Generator(device=dev).manual_seed(3)
    A = torch.randint(-3, 4, (k, m), generator=g, device=dev).to(torch.float64)
    B = torch.randint(-3, 4, (k, n), generator=g, device=dev).to(torch.float64)
    want = A.T @ B  # exact as well (every partial sum is an integer below 2^53)
    C1 = _tn(L, torch, dev, A, B)
    assert torch.equal(C1, want)
    assert rel_err(C1[:3, :5].cpu().numpy(), A[:, :3].cpu().numpy().T @ B[:, :5].cpu().numpy()) == 0
    C2 = _tn(L, torch, dev, A, B)
    assert torch.equal(C1, C2)


def test_dgemm_nt_against_numpy(world, dev):
    """C (m x n) = A B^T and C += A B^T for ragged shapes, including far more output tiles than CTAs."""
    import torch
    from distributed_sddmm_b200 import lib
    L = lib()
    st = torch.cuda.current_stream().cuda_stream
    rng = np.random.default_rng(22)
    for m, n, k in ((70, 11, 19), (1, 1, 1), (64, 64, 16), (300, 130, 37), (5, 200, 3), (100000, 300, 64)):
        A, B = rng.uniform(-1, 1, (m, k)), rng.uniform(-1, 1, (n, k))
        C0 = rng.uniform(-1, 1, (m, n))
        dA, dB = torch.from_numpy(A).to(dev), torch.from_numpy(B).to(dev)
        dC = torch.full((m, n), float("nan"), dtype=torch.float64, device=dev)
        D.check(L.hnh_dgemm_nt_f64(dC.data_ptr(), dA.data_ptr(), dB.data_ptr(), m, n, k, 0, st))
        torch.cuda.synchronize()
        assert rel_err(dC.cpu().numpy(), A @ B.T) < 1e-13, (m, n, k)
        dC = torch.from_numpy(C0).to(dev)
        D.check(L.hnh_dgemm_nt_f64(dC.data_ptr(), dA.data_ptr(), dB.data_ptr(), m, n, k, 1, st))
        torch.cuda.synchronize()
        assert rel_err(dC.cpu().numpy(), C0 + A @ B.T) < 1e-13, (m, n, k)


def test_activation_derivatives_exact(world, dev):
    import torch
    from distributed_sddmm_b200 import lib
    L = lib()
    st = torch.cuda.current_stream().cuda_stream
    rng = np.random.default_rng(23)
    x = rng.uniform(-1, 1, 10007)
    x[::7] = 0.0
    dx = torch.from_numpy(x).to(dev)
    dy = torch.full_like(dx, float("nan"))
    D.check(L.hnh_leaky_relu_grad_f64(dy.data_ptr(), dx.data_ptr(), x.size, 0.25, st))
    assert np.array_equal(dy.cpu().numpy(), np.where(x > 0, 1.0, 0.25))
    D.check(L.hnh_leaky_relu_grad_f64(dx.data_ptr(), dx.data_ptr(), x.size, 0.25, st))  # in place
    assert np.array_equal(dx.cpu().numpy(), np.where(x > 0, 1.0, 0.25))
    grad = rng.uniform(-1, 1, (33, 17))
    out = np.maximum(rng.uniform(-1, 1, (33, 17)), 0.0)  # a ReLU output: zeros included
    dgrad, dout = torch.from_numpy(grad).to(dev), torch.from_numpy(out).to(dev)
    dst = torch.full((33, 5), float("nan"), dtype=torch.float64, device=dev)
    D.check(L.hnh_relu_cols_backward_f64(dst.data_ptr(), dgrad.data_ptr(), dout.data_ptr(), 17, 10, 33, 5, st))
    assert np.array_equal(dst.cpu().numpy(), np.where(out[:, 10:15] > 0, grad[:, 10:15], 0.0))


def _p1_net(name, logM=8, npr=6):
    N = 1 << logM
    rows, cols, _ = orc.er_tuples(logM, npr, SEED)
    layers, X0, weights = gat_inputs(N, LAYERS, SEED)
    S = D.SpmatLocal.load_er(logM, npr, SEED)
    alg = D.Algorithm(name, S, layers[0][0], 1)
    net = D.GAT(alg, layers, 0.2)
    for i, (_, _, heads) in enumerate(layers):
        for h in range(heads):
            net.set_weight(i, h, weights[i][h])
    net.set_input(X0)
    G = np.random.default_rng(SEED + 5).uniform(-1, 1, net.buffer_shape(len(layers)))
    return dict(N=N, rows=rows, cols=cols, layers=layers, X0=X0, weights=weights, S=S, alg=alg, net=net, G=G)


@pytest.mark.parametrize("name", ALGS)
def test_p1_gat_backward_matches_autograd(world, name):
    """Input gradient and every head's weight gradient of both layers against torch.autograd; the backward pass leaves
    the activations and the weights as they were."""
    P = _p1_net(name)
    net, layers = P["net"], P["layers"]
    net.forward()
    out_before = [net.buffer(i) for i in range(len(layers) + 1)]
    net.backward(P["G"])
    dX0, dW = gbo.gat_backward_global(P["rows"], P["cols"], P["N"], layers, P["weights"], 0.2, P["X0"], P["G"])
    assert np.abs(dX0).max() > 0
    assert rel_err(net.input_grad(), dX0) < 1e-10
    for i, (_, _, heads) in enumerate(layers):
        for h in range(heads):
            assert np.abs(dW[i][h]).max() > 0, (i, h)
            assert rel_err(net.weight_grad(i, h), dW[i][h]) < 1e-10, (name, i, h)
    for i in range(len(layers) + 1):
        assert np.array_equal(net.buffer(i), out_before[i]), i
    # the weights are untouched: a second forward pass reproduces the output bit for bit
    net.forward()
    assert np.array_equal(net.buffer(len(layers)), out_before[-1])


@pytest.mark.parametrize("name", ALGS)
def test_p1_gat_sgd_steps_track_autograd(world, name):
    """Three steps of W -= lr dW driven from Python (forward, backward, update, set_weight) follow the same three
    steps of the autograd model."""
    P = _p1_net(name)
    net, layers = P["net"], P["layers"]
    # the output is cubic in the weights per layer and the gradients are large: a step of about 1% of the weights
    _, dW0 = gbo.gat_backward_global(P["rows"], P["cols"], P["N"], layers, P["weights"], 0.2, P["X0"], P["G"])
    lr = 0.01 / max(np.abs(w).max() for per in dW0 for w in per)
    mine = [[w.copy() for w in per] for per in P["weights"]]
    ref_w = [[w.copy() for w in per] for per in P["weights"]]
    for step in range(3):
        net.forward()
        net.backward(P["G"])
        _, dW = gbo.gat_backward_global(P["rows"], P["cols"], P["N"], layers, ref_w, 0.2, P["X0"], P["G"])
        for i, (_, _, heads) in enumerate(layers):
            for h in range(heads):
                mine[i][h] = mine[i][h] - lr * net.weight_grad(i, h)
                net.set_weight(i, h, mine[i][h])
                ref_w[i][h] = ref_w[i][h] - lr * dW[i][h]
    for i, (_, _, heads) in enumerate(layers):
        for h in range(heads):
            assert rel_err(mine[i][h], ref_w[i][h]) < 1e-9, (name, i, h)
            assert np.abs(ref_w[i][h] - P["weights"][i][h]).max() > 1e-3 * np.abs(P["weights"][i][h]).max()  # they moved
    net.forward()
    want = gbo.gat_forward_global_torch(P["rows"], P["cols"], P["N"], layers, ref_w, 0.2, P["X0"])
    assert rel_err(net.buffer(len(layers)), want) < 1e-9


def test_p1_gat_backward_needs_a_current_forward_pass_and_the_output_shape(world):
    P = _p1_net("15d_fusion1", logM=6, npr=4)
    net = P["net"]
    with pytest.raises(RuntimeError, match="code -1.*no forward pass"):
        net.backward(P["G"])
    with pytest.raises(RuntimeError, match="code -1"):
        net.weight_grad(0, 0)  # nothing computed yet
    net.forward()
    net.backward(P["G"])
    net.set_weight(1, 2, P["weights"][1][2])
    with pytest.raises(RuntimeError, match="no forward pass"):
        net.backward(P["G"])
    net.forward()
    net.set_input(P["X0"])
    with pytest.raises(RuntimeError, match="no forward pass"):
        net.backward(P["G"])
    net.forward()
    net.backward(P["G"])
    with pytest.raises(ValueError):
        net.backward(P["G"][:, :-1])


def test_gat_train_benchmark_record(world):
    S = D.SpmatLocal.load_er(10, 8, SEED)
    rec = D.benchmark_algorithm(S, "15d_fusion1", R=32, c=1, fused=True, app="gat_train", trials=1, warmup=0)
    assert rec["overall_throughput"] > 0 and rec["elapsed"] > 0
