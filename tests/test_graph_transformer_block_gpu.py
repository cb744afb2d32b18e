"""Graph transformer blocks on the GPU on one rank: forward output, input gradient and every parameter gradient against
the fp64 model of tests/graph_transformer_block_oracle.py to a relative error of 1e-10, for 1-3 layers, ffn_ratio 1 and
2, every (gate, edge) combination and attention dropout 0 and 0.3; head widths 32, 64 and 256 and an odd width;
duplicate entries and empty rows on every algorithm at p = 1; a torch LayerNorm / Linear state dict loaded by
transposing; bit-identical repeats; ffn_ratio = 0 bit-identical to the model of the old constructor; refusals.  The
kernels alone are in tests/test_layer_norm_gpu.py, multi-rank cases in
tests/test_graph_transformer_block_multirank_gpu.py."""
import ctypes as C

import numpy as np
import pytest
import torch

from distributed_sddmm_b200 import driver as D
from distributed_sddmm_b200 import lib
from oracle import hnh_oracle as orc
from tests import graph_transformer_block_oracle as gbo
from tests import graph_transformer_oracle as gto
from tests.test_graph_transformer_gpu import attr_of, grad_err, rel_err
from tests.test_sparse_attention_bias import _pattern

pytestmark = pytest.mark.gpu
SEED = 0xC0FFEE + 83


@pytest.fixture(scope="module")
def world():
    D.world_init("self")
    yield
    D.world_finalize()


def build(layers, edge_dim, beta, ffn, logM=7, npr=5, alg_name="15d_fusion1", pattern=None, seed=SEED, eps=1e-5):
    N = 1 << logM
    if pattern is None:
        rows, cols, _ = orc.er_tuples(logM, npr, seed)
    else:
        rows, cols = pattern
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    S = D.SpmatLocal.from_tuples(N, N, rows, cols, np.ones(len(rows)))
    alg = D.Algorithm(alg_name, S, layers[0][0], 1)
    net = D.GraphTransformer(alg, layers, edge_dim=edge_dim, beta=beta, ffn_ratio=ffn, norm_eps=eps)
    rng = np.random.default_rng(seed + 1)
    params = gbo.random_params(layers, edge_dim, beta, ffn, rng)
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
                attr=attr_of(rows, cols, edge_dim) if edge_dim else None, beta=beta, eps=eps)


def check_against_model(P, dropout, seed):
    net, N, layers = P["net"], P["N"], P["layers"]
    net.forward(dropout, seed)
    args = (P["rows"], P["cols"], N, layers, P["params"], P["X"])
    kw = dict(attr=P["attr"], beta=P["beta"], p=dropout, seed=seed, eps=P["eps"])
    want = gbo.forward_np(*args, **kw)
    out = net.buffer(len(layers))[:N]
    assert np.abs(want).max() > 0
    assert rel_err(out, want) < 1e-10
    net.backward(P["G"])
    dX, dP = gbo.backward_np(*args, P["G"][:N], **kw)
    assert rel_err(net.input_grad()[:N], dX) < 1e-10
    for l, grads in enumerate(dP):
        scale = max(np.abs(g).max() for g in grads.values())
        assert sorted(grads) == sorted(net.param_names())
        for name, g in grads.items():
            got = net.param_grad(l, name)
            assert got.shape == g.shape, (l, name)
            assert grad_err(got, g, scale) < 1e-10, (l, name, grad_err(got, g, scale))


LAYER_SETS = {1: [(6, 4, 2)], 2: [(6, 4, 2), (8, 3, 3)], 3: [(6, 4, 2), (8, 3, 3), (9, 8, 1)]}


@pytest.mark.parametrize("dropout", [0.0, 0.3])
@pytest.mark.parametrize("beta", [False, True])
@pytest.mark.parametrize("edge_dim", [0, 3])
@pytest.mark.parametrize("ffn", [1, 2])
@pytest.mark.parametrize("n_layers", [1, 2, 3])
def test_block_matches_model(world, n_layers, ffn, edge_dim, beta, dropout):
    P = build(LAYER_SETS[n_layers], edge_dim, beta, ffn)
    check_against_model(P, dropout, 17)


@pytest.mark.parametrize("d", [32, 64, 256, 5])
def test_block_head_widths(world, d):
    """r = 64, 128, 256 and an odd width (r = 15: the scalar LayerNorm and bias paths), hidden width 2r."""
    H = 3 if d == 5 else 2 if d < 256 else 1
    P = build([(7, d, H), (d * H, 4, 2)], 2, True, 2, logM=6)
    check_against_model(P, 0.3, 5)


@pytest.mark.parametrize("alg_name", ["15d_fusion1", "15d_fusion2", "15d_sparse", "25d_dense_replicate", "25d_sparse_replicate"])
def test_block_duplicates_and_empty_rows(world, alg_name):
    rng = np.random.default_rng(13)
    rows, cols = _pattern(rng, 64, 64, per_row=6)
    rows, cols = np.concatenate([rows, [5, 5, 5]]), np.concatenate([cols, [9, 9, 9]])
    P = build(LAYER_SETS[2], 3, True, 1, logM=6, alg_name=alg_name, pattern=(rows, cols), eps=1e-3)
    check_against_model(P, 0.3, 23)


def test_torch_state_dict_maps_on(world):
    """norm1 / lin1 / lin2 / norm2 of a torch model load by transposing the Linear weights and give its outputs."""
    layers = [(6, 4, 2), (8, 3, 2)]
    P = build(layers, 0, False, 2, logM=6)
    net, N = P["net"], P["N"]
    torch.manual_seed(3)
    mods = []
    for l, (f, d, H) in enumerate(layers):
        r = d * H
        m = dict(norm1=torch.nn.LayerNorm(r).double(), lin1=torch.nn.Linear(r, 2 * r).double(),
                 lin2=torch.nn.Linear(2 * r, r).double(), norm2=torch.nn.LayerNorm(r).double())
        with torch.no_grad():
            for k in ("norm1", "norm2"):
                m[k].weight.uniform_(0.5, 1.5)
                m[k].bias.uniform_(-0.5, 0.5)
        sd = {k: v.detach().numpy() for k, v in ((f"{a}.{b}", t) for a, mod in m.items() for b, t in mod.state_dict().items())}
        net.set_param(l, "norm1", sd["norm1.weight"])
        net.set_param(l, "norm1_bias", sd["norm1.bias"])
        net.set_param(l, "ffn1", np.vstack([sd["lin1.weight"].T, sd["lin1.bias"]]))
        net.set_param(l, "ffn2", np.vstack([sd["lin2.weight"].T, sd["lin2.bias"]]))
        net.set_param(l, "norm2", sd["norm2.weight"])
        net.set_param(l, "norm2_bias", sd["norm2.bias"])
        mods.append(m)
    net.forward()
    x = gto._t(P["X"])
    with torch.no_grad():
        for l, lay in enumerate(layers):
            tp = {k: gto._t(v) for k, v in P["params"][l].items()}
            h = mods[l]["norm1"](gto.model_torch(P["rows"], P["cols"], N, [lay], [tp], x))
            x = mods[l]["norm2"](h + mods[l]["lin2"](torch.relu(mods[l]["lin1"](h))))
    assert rel_err(net.buffer(len(layers))[:N], x.numpy()) < 1e-10


def test_block_backward_repeats_bit_identical(world):
    P = build(LAYER_SETS[3], 3, True, 2)
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


def _block_handle(alg, layers, ffn, eps, edge_dim=0, beta=0):
    flat = (C.c_int * (3 * len(layers)))(*[x for l in layers for x in l])
    h = C.c_void_p()
    rc = lib().hnhd_gt_create_block(alg.h, len(layers), flat, edge_dim, beta, ffn, eps, C.byref(h))
    return rc, h


def test_ffn_ratio_zero_is_the_old_model_bit_for_bit(world):
    """hnhd_gt_create_block with ffn_ratio = 0 (and any valid eps) gives the bits of hnhd_gt_create: outputs, the input
    gradient and every parameter gradient."""
    old = build(LAYER_SETS[3], 3, True, 0)
    net_old, layers = old["net"], old["layers"]
    rc, h = _block_handle(old["alg"], layers, 0, 0.25, 3, 1)
    assert rc == 0
    new = D.GraphTransformer.__new__(D.GraphTransformer)
    new.alg, new.h, new.layers, new.edge_dim, new.beta, new.ffn_ratio = old["alg"], h, layers, 3, True, 0
    assert new.param_names() == net_old.param_names()
    for l, Pl in enumerate(old["params"]):
        for name, v in Pl.items():
            new.set_param(l, name, v)
    new.set_input(np.vstack([old["X"], np.zeros((net_old.buffer_shape(0)[0] - old["N"], layers[0][0]))]))
    alg = old["alg"]
    new.set_edge_attributes(attr_of(*alg.entry_coordinates("A"), 3), attr_of(*alg.entry_coordinates("B"), 3))
    for net in (net_old, new):
        net.forward(0.3, 7)
        net.backward(old["G"])
    assert np.array_equal(net_old.buffer(len(layers)), new.buffer(len(layers)))
    assert np.array_equal(net_old.input_grad(), new.input_grad())
    for l in range(len(layers)):
        for name in net_old.param_names():
            assert np.array_equal(net_old.param_grad(l, name), new.param_grad(l, name)), (l, name)
    for name in gbo.BLOCK:
        with pytest.raises(RuntimeError, match="code -1.*no parameter"):
            new.param_shape(0, name)


def test_block_arguments_are_refused(world):
    N = 64
    rows, cols, _ = orc.er_tuples(6, 4, SEED)
    S = D.SpmatLocal.from_tuples(N, N, rows, cols, np.ones(len(rows)))
    alg = D.Algorithm("15d_fusion1", S, 6, 1)
    layers = [(6, 4, 2), (8, 3, 3)]
    assert _block_handle(alg, layers, -1, 1e-5)[0] == -1 and b"ffn_ratio" in lib().hnh_last_error_string()
    for bad in (0.0, -1.0, float("nan"), float("inf")):
        assert _block_handle(alg, layers, 2, bad)[0] == -1 and b"norm_eps" in lib().hnh_last_error_string()
    plain = D.GraphTransformer(alg, layers)
    for name in gbo.BLOCK:
        with pytest.raises(RuntimeError, match="code -1.*no parameter"):
            plain.param_shape(0, name)
    net = D.GraphTransformer(alg, layers, ffn_ratio=3)
    assert net.param_names()[-6:] == list(gbo.BLOCK)
    for l, r in ((0, 8), (1, 9)):
        h = 3 * r
        assert net.param_shape(l, "norm1") == (r,) and net.param_shape(l, "norm1_bias") == (r,)
        assert net.param_shape(l, "norm2") == (r,) and net.param_shape(l, "norm2_bias") == (r,)
        assert net.param_shape(l, "ffn1") == (r + 1, h) and net.param_shape(l, "ffn2") == (h + 1, r)
        assert np.array_equal(net.param(l, "norm1"), np.ones(r)) and np.array_equal(net.param(l, "norm2"), np.ones(r))
        assert not net.param(l, "ffn1").any() and not net.param(l, "norm2_bias").any()
    with pytest.raises(ValueError):
        net.set_param(0, "ffn1", np.zeros((24, 9)))
    # the block parameters make the activations stale too
    net.set_input(np.ones(net.buffer_shape(0)))
    net.forward()
    G = np.ones(net.buffer_shape(2))
    net.backward(G)
    net.set_param(1, "ffn2", np.full((28, 9), 0.1))
    with pytest.raises(RuntimeError, match="no forward pass"):
        net.backward(G)
    net.forward()
    net.backward(G)


def test_graph_transformer_block_benchmark_records(world):
    S = D.SpmatLocal.load_er(10, 8, SEED)
    for app in ("graph_transformer_block", "graph_transformer_block_train"):
        rec = D.benchmark_algorithm(S, "15d_fusion1", R=256, c=1, fused=True, app=app, trials=1, warmup=0)
        assert rec["overall_throughput"] > 0 and rec["elapsed"] > 0
