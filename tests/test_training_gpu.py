"""Training on the GPU on one rank.  The kernels alone against torch: hnh_cross_entropy_f64 (C from 1 to past the register
table, logits up to +-1000 with exact ties, every row ignored, odd ld and misaligned rows, more rows than one resident
wave, bit-identical repeats) and hnh_adamw_f64 (5 steps, odd and misaligned tensors, weight decay 0 and 0.01, with and
without a clip coefficient).  The models: five train steps of the graph transformer (without and with blocks, gate and
edge features, dropout) and of GAT with each attention kind against tests/training_oracle.py, an lr schedule and
clipping, refusals, and a convergence run on a learnable task.  Multi-rank cases are in
tests/test_training_multirank_gpu.py."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from distributed_sddmm_b200 import driver as D
from distributed_sddmm_b200 import lib
from oracle import hnh_oracle as orc
from tests import gat_additive_oracle as gao
from tests import gatv2_oracle as gv2
from tests import graph_transformer_block_oracle as gbo
from tests import training_oracle as tro
from tests.test_graph_transformer_gpu import attr_of

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
SEED = 0xC0FFEE + 131


@pytest.fixture(scope="module")
def world():
    D.world_init("self")
    yield
    D.world_finalize()


def _st():
    return torch.cuda.current_stream().cuda_stream


# ---- hnh_cross_entropy_f64 ------------------------------------------------------------------------------------------
def cross_entropy(x, labels, ld=None, offset=0, inv=None):
    """Runs the kernel on host logits x (n x C) stored with leading dimension ld at `offset` doubles into a buffer;
    returns (dlogits n x C, sums)."""
    n, C = x.shape
    ld = ld or C
    buf = torch.full((offset + n * ld + 1,), math.nan, dtype=torch.float64, device=DEV)
    rows = buf[offset:offset + n * ld].view(n, ld)
    rows[:, :C] = torch.from_numpy(x).to(DEV)
    dbuf = torch.full_like(buf, math.nan)
    lab = torch.from_numpy(np.asarray(labels, np.int32)).to(DEV)
    sums = torch.full((2,), math.nan, dtype=torch.float64, device=DEV)
    nbytes = lib().hnh_cross_entropy_workspace_bytes(n)
    ws = torch.empty(nbytes // 8 + 1, dtype=torch.float64, device=DEV)
    labelled = int(((np.asarray(labels) >= 0) & (np.asarray(labels) < C)).sum())
    inv = (1.0 / labelled if labelled else 0.0) if inv is None else inv
    rc = lib().hnh_cross_entropy_f64(dbuf.data_ptr() + 8 * offset, sums.data_ptr(), buf.data_ptr() + 8 * offset, lab.data_ptr(),
                                     n, C, ld, inv, ws.data_ptr(), nbytes, _st())
    assert rc == 0, lib().hnh_last_error_string()
    torch.cuda.synchronize()
    d = dbuf[offset:offset + n * ld].view(n, ld)
    if ld > C:
        assert torch.isnan(d[:, C:]).all()  # the columns past C are not written
    return d[:, :C].cpu().numpy(), sums.cpu().numpy()


def ce_reference(x, labels):
    lab = torch.from_numpy(np.where(np.asarray(labels) < 0, -1, np.asarray(labels)).astype(np.int64))
    xt = torch.from_numpy(x).requires_grad_()
    m = lab >= 0
    total = F.cross_entropy(xt, lab, ignore_index=-1, reduction="sum")
    total.backward()
    correct = int((xt.detach().argmax(1)[m] == lab[m]).sum())
    k = int(m.sum())
    return xt.grad.numpy() / k if k else np.zeros_like(x), float(total), correct


def check_ce(x, labels, **kw):
    d, sums = cross_entropy(x, labels, **kw)
    dw, loss, correct = ce_reference(x, labels)
    assert abs(sums[0] - loss) <= 1e-13 * max(abs(loss), 1.0), (sums[0], loss)
    assert sums[1] == correct
    assert np.abs(d - dw).max() <= 1e-13 * max(np.abs(dw).max(), 1e-300) or not dw.any() and not d.any()
    return d, sums


@pytest.mark.parametrize("C", [1, 2, 3, 40, 64, 255, 256, 1024, 1536, 1601])
def test_cross_entropy_matches_torch(world, C):
    rng = np.random.default_rng(C)
    n = 257
    x = rng.uniform(-1000, 1000, (n, C))
    x[::3] = np.round(x[::3] / 250) * 250  # exact ties, the argmax goes to the lowest index
    x[1::7] = rng.standard_normal((len(x[1::7]), C))
    labels = rng.integers(-2, C, n)
    labels[5] = -1
    check_ce(x, labels)
    d1, s1 = cross_entropy(x, labels)
    d2, s2 = cross_entropy(x, labels)
    assert np.array_equal(d1, d2) and np.array_equal(s1, s2)


@pytest.mark.parametrize("C", [3, 40, 256, 1536, 1601])
def test_cross_entropy_odd_ld_and_misaligned_rows(world, C):
    rng = np.random.default_rng(C + 1)
    x = rng.uniform(-30, 30, (129, C))
    labels = rng.integers(-1, C, 129)
    for ld, offset in ((C + 1, 0), (C, 1), (C + 3, 1), (C + 2, 0)):
        check_ce(x, labels, ld=ld, offset=offset)


def test_cross_entropy_all_rows_ignored(world):
    x = np.random.default_rng(3).uniform(-5, 5, (100, 40))
    d, sums = cross_entropy(x, -np.ones(100, np.int64))
    assert not d.any() and not sums.any()
    # labels at or past C are ignored too, and never read
    d, sums = cross_entropy(x, np.full(100, 40), inv=0.5)
    assert not d.any() and not sums.any()


@pytest.mark.parametrize("C,n", [(40, 30000), (256, 12000), (1536, 2500)])
def test_cross_entropy_past_one_wave(world, C, n):
    rng = np.random.default_rng(n)
    x = rng.standard_normal((n, C)) * 4
    labels = rng.integers(-1, C, n)
    check_ce(x, labels)


# ---- hnh_adamw_f64 --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2, 3, 1000, (1 << 20) + 1])
@pytest.mark.parametrize("wd", [0.0, 0.01])
@pytest.mark.parametrize("clip", [None, 0.37])
@pytest.mark.parametrize("offset", [0, 1])
def test_adamw_matches_torch(world, n, wd, clip, offset):
    if n > 1000 and offset and clip is None:
        pytest.skip("the large size runs misaligned with a clip coefficient")
    rng = np.random.default_rng(n + offset)
    p0 = rng.standard_normal(n)
    lr, b1, b2, eps = 3e-2, 0.9, 0.999, 1e-8
    bufs = [torch.zeros(n + offset + 1, dtype=torch.float64, device=DEV) for _ in range(4)]
    P, M, V, G = (b[offset:offset + n] for b in bufs)
    P.copy_(torch.from_numpy(p0))
    coef = torch.tensor([clip if clip else 1.0], dtype=torch.float64, device=DEV)
    tp = torch.tensor(p0, requires_grad=True)
    opt = torch.optim.AdamW([tp], lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd, foreach=False)
    for t in range(1, 6):
        g = rng.standard_normal(n) * (10.0 ** rng.integers(-3, 3))
        G.copy_(torch.from_numpy(g))
        rc = lib().hnh_adamw_f64(P.data_ptr(), M.data_ptr(), V.data_ptr(), G.data_ptr(), n, lr, b1, b2, eps, wd, 1 - b1 ** t,
                                 1 - b2 ** t, coef.data_ptr() if clip else None, _st())
        assert rc == 0, lib().hnh_last_error_string()
        tp.grad = torch.from_numpy(g * clip if clip else g)
        opt.step()
    torch.cuda.synchronize()
    want = tp.detach().numpy()
    assert np.abs(P.cpu().numpy() - want).max() <= 1e-13 * np.abs(want).max()
    st = opt.state[tp]
    assert np.abs(M.cpu().numpy() - st["exp_avg"].numpy()).max() <= 1e-13 * np.abs(st["exp_avg"].numpy()).max()
    assert np.abs(V.cpu().numpy() - st["exp_avg_sq"].numpy()).max() <= 1e-13 * np.abs(st["exp_avg_sq"].numpy()).max()
    assert np.array_equal(G.cpu().numpy(), g)  # grad is not written


# ---- the models ------------------------------------------------------------------------------------------------------
def _graph(logM, npr, seed):
    rows, cols, _ = orc.er_tuples(logM, npr, seed)
    return np.asarray(rows, np.int64), np.asarray(cols, np.int64)


def _labels(rng, n_rows, N, C):
    lab = rng.integers(0, C, n_rows)
    lab[rng.random(n_rows) < 0.2] = -1
    lab[N:] = -1
    return lab


def _close(got, want, tol):
    return np.abs(got - want).max() <= tol * max(np.abs(want).max(), 1.0)


def check_steps(got, want):
    for t, (g, w) in enumerate(zip(got, want)):
        assert abs(g.loss - w[0]) <= 1e-10 * abs(w[0]), (t, g, w)
        assert (g.correct, g.labelled) == (w[1], w[2]), (t, g, w)
        assert abs(g.grad_norm - w[3]) <= 1e-10 * abs(w[3]), (t, g, w)


GT_CASES = {
    "plain": dict(layers=[(6, 4, 2), (8, 5, 1)], edge_dim=0, beta=False, ffn=0, dropout=0.0),
    "blocks": dict(layers=[(6, 4, 2), (8, 5, 1)], edge_dim=0, beta=False, ffn=2, dropout=0.0),
    "gate_edge": dict(layers=[(6, 4, 2), (8, 3, 2)], edge_dim=3, beta=True, ffn=0, dropout=0.0),
    "dropout": dict(layers=[(6, 4, 2), (8, 5, 1)], edge_dim=2, beta=True, ffn=1, dropout=0.3),
}


@pytest.mark.parametrize("name", sorted(GT_CASES))
def test_graph_transformer_train_steps_match_torch(world, name):
    cfg, steps, N = GT_CASES[name], 5, 128
    layers, edge_dim, beta, ffn = cfg["layers"], cfg["edge_dim"], cfg["beta"], cfg["ffn"]
    rows, cols = _graph(7, 5, SEED)
    S = D.SpmatLocal.from_tuples(N, N, rows, cols, np.ones(len(rows)))
    alg = D.Algorithm("15d_fusion1", S, layers[0][0], 1)
    net = D.GraphTransformer(alg, layers, edge_dim=edge_dim, beta=beta, ffn_ratio=ffn)
    rng = np.random.default_rng(SEED + len(name))
    params = gbo.random_params(layers, edge_dim, beta, ffn, rng)
    for l, P in enumerate(params):
        for k, v in P.items():
            net.set_param(l, k, v)
    X = rng.uniform(-1, 1, (N, layers[0][0]))
    net.set_input(np.vstack([X, np.zeros((net.buffer_shape(0)[0] - N, X.shape[1]))]))
    if edge_dim:
        net.set_edge_attributes(attr_of(*alg.entry_coordinates("A"), edge_dim), attr_of(*alg.entry_coordinates("B"), edge_dim))
    C = layers[-1][1] * layers[-1][2]
    lab = _labels(rng, net.buffer_shape(len(layers))[0], N, C)
    labels = D.NodeLabels(net, lab, C)
    lrs = [1e-2, 2e-2, 3e-2, 2e-2, 1e-2] if name == "plain" else [1e-2] * steps
    clip = 0.05 if name in ("plain", "gate_edge") else None
    opt = D.AdamW(lr=lrs[0], weight_decay=0.01, max_grad_norm=clip)
    seeds = [11 + 7 * t for t in range(steps)]
    got = []
    for t in range(steps):
        opt.lr = lrs[t]
        got.append(net.train_step(labels, opt, cfg["dropout"], seeds[t]))
    want, tparams = tro.train_gt(rows, cols, N, layers, params, X, lab[:N], steps, attr=attr_of(rows, cols, edge_dim) if edge_dim else None,
                                 beta=beta, ffn=ffn, dropout=cfg["dropout"], seeds=seeds, lr=lrs[0], lrs=lrs, weight_decay=0.01,
                                 max_grad_norm=clip)
    check_steps(got, want)
    if clip:
        assert any(w[3] > clip for w in want)  # clipping was active
    for l, P in enumerate(tparams):
        for k, w in P.items():
            g = net.param(l, k)
            if k == "key_bias":  # its gradient is rounding noise on both sides; Adam turns it into steps of up to lr
                assert np.abs(g - w).max() <= sum(lrs) * 1.01, (l, k)
            else:
                assert _close(g, w, 1e-9), (name, l, k, np.abs(g - w).max())


@pytest.mark.parametrize("kind", ["leaky", "softmax", "additive", "gatv2"])
def test_gat_train_steps_match_torch(world, kind):
    steps, N = 5, 128
    layers = [(8, 4, 2), (8, 6, 1)]
    rows, cols = _graph(7, 5, SEED + 1)
    S = D.SpmatLocal.from_tuples(N, N, rows, cols, np.ones(len(rows)))
    alg = D.Algorithm("15d_fusion1", S, layers[0][0], 1)
    net = D.GAT(alg, layers, attention=kind)
    rng = np.random.default_rng(SEED + 2)
    weights = [[rng.uniform(-1, 1, (f, d)) / math.sqrt(f) for _ in range(H)] for f, d, H in layers]
    a1, a2 = gao.attention_inputs(layers, SEED) if kind != "gatv2" else (gv2.attention_inputs(layers, SEED),) * 2
    for l, (f, d, H) in enumerate(layers):
        for h in range(H):
            net.set_weight(l, h, weights[l][h])
            net.set_attention_vectors(l, h, a1[l][h], a2[l][h])
    X = rng.uniform(0, 1, (N, layers[0][0]))
    net.set_input(np.vstack([X, np.zeros((net.buffer_shape(0)[0] - N, X.shape[1]))]))
    C = 6
    lab = _labels(rng, net.buffer_shape(len(layers))[0], N, C)
    labels = D.NodeLabels(net, lab, C)
    opt = D.AdamW(lr=1e-2)
    got = [net.train_step(labels, opt) for _ in range(steps)]
    want, ws, u1, u2 = tro.train_gat(kind, rows, cols, N, layers, weights, a1, a2, X, lab[:N], steps, lr=1e-2)
    check_steps(got, want)
    for l, (f, d, H) in enumerate(layers):
        for h in range(H):
            assert _close(net.weight(l, h), ws[l][h], 1e-9), (kind, l, h)
            v1, v2 = net.attention_vectors(l, h)
            assert _close(v1, u1[l][h], 1e-9) and _close(v2, u2[l][h], 1e-9), (kind, l, h)
    if kind in ("leaky", "softmax"):  # a1, a2 unread: decay alone, (1 - lr wd)^t
        v1, _ = net.attention_vectors(0, 0)
        assert np.allclose(v1, np.asarray(a1[0][0]) * (1 - 1e-2 * 1e-2) ** steps, rtol=1e-14, atol=0)


# ---- convergence -----------------------------------------------------------------------------------------------------
def test_graph_transformer_learns_a_neighbourhood_task(world):
    """Labels are a fixed function of the neighbours' mean features; 100 steps halve the loss and lift the accuracy well
    above chance."""
    N, f, C = 256, 8, 4
    rows, cols = _graph(8, 6, SEED + 5)
    rng = np.random.default_rng(SEED + 6)
    X = rng.standard_normal((N, f))
    deg = np.bincount(rows, minlength=N)
    mean = np.zeros((N, f))
    np.add.at(mean, rows, X[cols])
    mean /= np.maximum(deg, 1)[:, None]
    lab = np.argmax(mean @ rng.standard_normal((f, C)), 1)
    lab[deg == 0] = -1
    S = D.SpmatLocal.from_tuples(N, N, rows, cols, np.ones(len(rows)))
    alg = D.Algorithm("15d_fusion2", S, f, 1)
    net = D.GraphTransformer(alg, [(f, 8, 2), (16, C, 1)])
    params = gbo.random_params([(f, 8, 2), (16, C, 1)], 0, False, 0, rng, scale=0.3)
    for l, P in enumerate(params):
        for k, v in P.items():
            net.set_param(l, k, v)
    net.set_input(np.vstack([X, np.zeros((net.buffer_shape(0)[0] - N, f))]))
    labels = D.NodeLabels(net, np.concatenate([lab, -np.ones(net.buffer_shape(2)[0] - N, np.int64)]), C)
    opt = D.AdamW(lr=2e-2, weight_decay=0.0)
    hist = [net.train_step(labels, opt) for _ in range(100)]
    assert hist[-1].loss < 0.5 * hist[0].loss, (hist[0], hist[-1])
    assert hist[-1].correct / hist[-1].labelled > 0.6, hist[-1]
