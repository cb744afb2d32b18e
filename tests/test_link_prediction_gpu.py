"""Link prediction on the GPU on one rank.  The kernel hnh_link_bce_f64 against torch: the table widths and others from
r = 1 to 257, odd leading dimensions and misaligned rows, rows without entries, duplicates and a hub row (and the skewed
graph of tests/skewed_graph.py), targets 0, 1 and 0.25 with |s| up to 1e3, a pre-filled dX and stats that are added
to, every nullable output null, more rows than one resident wave, bit-identical repeats.  The op
Distributed_Sparse::linkLoss at p = 1 under every algorithm name; refusals; five link train steps of the graph
transformer and of GAT with each attention kind against tests/link_prediction_oracle.py; link_evaluate's scores; and a
convergence run on a stochastic block model with a held-out AUC.  Multi-rank cases are in
tests/test_link_prediction_multirank_gpu.py."""
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
from tests import link_prediction_oracle as lpo
from tests.skewed_graph import skewed_tuples
from tests.test_graph_transformer_gpu import attr_of

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
SEED = 0xC0FFEE + 171
ALGS = ["15d_fusion1", "15d_fusion2", "15d_sparse", "25d_dense_replicate", "25d_sparse_replicate"]


@pytest.fixture(scope="module")
def world():
    D.world_init("self")
    yield
    D.world_finalize()


def _st():
    return torch.cuda.current_stream().cuda_stream


# ---- hnh_link_bce_f64 -----------------------------------------------------------------------------------------------
def csr_block(rng, n, m, per_row=6, hub=True):
    """A CSR block of n rows over m columns: a third of the rows empty, duplicated columns, a hub row of m / 2 entries."""
    deg = rng.integers(1, per_row + 1, n)
    deg[rng.random(n) < 0.33] = 0
    if hub and n > 3:
        deg[3] = m // 2
    cols = [np.sort(rng.integers(0, m, d)) for d in deg]
    for c in cols[1::5]:
        if len(c) > 1:
            c[1] = c[0]  # a duplicate
    rowStart = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    return rowStart, np.concatenate(cols).astype(np.int64) if n else np.zeros(0, np.int64)


def operands(rng, n, m, r, nnz):
    X = rng.standard_normal((n, r)) / r ** 0.25
    Y = rng.standard_normal((m, r)) / r ** 0.25
    X[rng.random(n) < 0.1] *= 300.0  # scores up to about 1e3
    y = rng.choice([0.0, 1.0, 0.25], nnz)
    return X, Y, y


def _dev_rows(A, ld, offset):
    """A (rows x r) as a device buffer with leading dimension ld, starting `offset` doubles in; NaN elsewhere."""
    n, r = A.shape
    buf = torch.full((offset + max(n * ld, 1) + 1,), math.nan, dtype=torch.float64, device=DEV)
    if n:
        buf[offset:offset + n * ld].view(n, ld)[:, :r] = torch.from_numpy(A).to(DEV)
    return buf


def run_bce(rowStart, col_idx, y, X, Y, inv, dX0=None, stats0=None, scores=True, ld=(None, None, None), offset=0):
    """Runs the kernel; returns (dX, stats, scores) as numpy (None where the output was null)."""
    n, r = X.shape
    ldx, ldy, lddx = (l or r for l in ld)
    xb, yb = _dev_rows(X, ldx, offset), _dev_rows(Y, ldy, offset)
    rs, ci = torch.from_numpy(rowStart).to(DEV), torch.from_numpy(col_idx).to(DEV)
    t = torch.from_numpy(np.asarray(y, np.float64)).to(DEV)
    db = _dev_rows(dX0, lddx, offset) if dX0 is not None else None
    sb = torch.from_numpy(stats0.copy()).to(DEV) if stats0 is not None else None
    sc = torch.full((len(col_idx) + 1,), math.nan, dtype=torch.float64, device=DEV) if scores else None
    p = lambda b, off=0: b.data_ptr() + 8 * off if b is not None else None  # noqa: E731
    rc = lib().hnh_link_bce_f64(rs.data_ptr(), ci.data_ptr(), t.data_ptr(), n, len(col_idx), p(xb, offset), ldx, p(yb, offset),
                                ldy, r, inv, p(db, offset), lddx, p(sb), 2, p(sc), _st())
    assert rc == 0, lib().hnh_last_error_string()
    torch.cuda.synchronize()
    dX = None
    if db is not None:
        d = db[offset:offset + n * lddx].view(n, lddx)
        if lddx > r:
            assert torch.isnan(d[:, r:]).all()  # the columns past r are not written
        dX = d[:, :r].cpu().numpy()
    if sc is not None:
        assert torch.isnan(sc[-1])
    return dX, sb.cpu().numpy() if sb is not None else None, sc[:-1].cpu().numpy() if sc is not None else None


def ref_bce(rowStart, col_idx, y, X, Y, inv, dX0, stats0):
    rows = np.repeat(np.arange(len(rowStart) - 1), np.diff(rowStart))
    s = (X[rows] * Y[col_idx]).sum(1)
    st, yt = torch.from_numpy(s), torch.from_numpy(np.asarray(y, np.float64))
    loss = F.binary_cross_entropy_with_logits(st, yt, reduction="none").numpy()
    g = (torch.sigmoid(st) - yt).numpy() * inv
    dX = dX0.copy()
    np.add.at(dX, rows, g[:, None] * Y[col_idx])
    stats = stats0.copy()
    np.add.at(stats[:, 0], rows, loss)
    np.add.at(stats[:, 1], rows, ((s > 0) == (np.asarray(y) > 0.5)).astype(np.float64))
    bound = (np.abs(X[rows]) * np.abs(Y[col_idx])).sum(1)  # the dot's rounding scale
    return dX, stats, s, bound


def check_bce(rowStart, col_idx, y, X, Y, inv=1e-2, **kw):
    rng = np.random.default_rng(len(col_idx))
    dX0, stats0 = rng.standard_normal(X.shape), rng.standard_normal((X.shape[0], 2))
    stats0[:, 1] = rng.integers(0, 5, len(stats0))  # counts stay exact whatever the order of the additions
    dX, stats, s = run_bce(rowStart, col_idx, y, X, Y, inv, dX0, stats0, **kw)
    wdX, wstats, ws, bound = ref_bce(rowStart, col_idx, y, X, Y, inv, dX0, stats0)
    assert np.isfinite(dX).all() and np.isfinite(stats).all()
    assert (np.abs(s - ws) <= 1e-13 * bound + 1e-300).all()
    assert np.abs(dX - wdX).max() <= 1e-12 * max(np.abs(wdX).max(), 1.0)
    assert np.abs(stats[:, 0] - wstats[:, 0]).max() <= 1e-12 * max(np.abs(wstats[:, 0]).max(), 1.0)
    near0 = np.zeros(len(stats), bool)  # rows with a score within rounding of 0 may count differently
    rows = np.repeat(np.arange(len(rowStart) - 1), np.diff(rowStart))
    np.logical_or.at(near0, rows, np.abs(ws) <= 1e-12 * bound)
    assert np.array_equal(stats[~near0, 1], wstats[~near0, 1])
    empty = np.diff(rowStart) == 0  # untouched rows
    assert np.array_equal(dX[empty], dX0[empty]) and np.array_equal(stats[empty], stats0[empty])
    return dX0, stats0, (dX, stats, s)


WIDTHS = [1, 3, 4, 8, 31, 64, 128, 255, 256, 257]


@pytest.mark.parametrize("r", WIDTHS)
def test_link_kernel_matches_torch(world, r):
    rng = np.random.default_rng(SEED + r)
    rowStart, col_idx = csr_block(rng, 300, 400)
    X, Y, y = operands(rng, 300, 400, r, len(col_idx))
    assert np.abs((X[np.repeat(np.arange(300), np.diff(rowStart))] * Y[col_idx]).sum(1)).max() > 100
    dX0, stats0, first = check_bce(rowStart, col_idx, y, X, Y)
    again = run_bce(rowStart, col_idx, y, X, Y, 1e-2, dX0, stats0)
    for a, b in zip(first, again):
        assert np.array_equal(a, b)  # bit-identical repeats


@pytest.mark.parametrize("r", [3, 4, 64, 256, 257])
def test_link_kernel_odd_ld_and_misaligned_rows(world, r):
    rng = np.random.default_rng(SEED + 2 * r)
    rowStart, col_idx = csr_block(rng, 200, 150)
    X, Y, y = operands(rng, 200, 150, r, len(col_idx))
    for ld, offset in (((r + 1, r, r), 0), ((r, r + 1, r), 0), ((r, r, r + 1), 0), ((r, r, r), 1), ((r + 3, r + 2, r + 1), 1)):
        check_bce(rowStart, col_idx, y, X, Y, ld=ld, offset=offset)


def test_link_kernel_nullable_outputs(world):
    rng = np.random.default_rng(SEED + 5)
    rowStart, col_idx = csr_block(rng, 120, 120)
    for r in (64, 7):
        X, Y, y = operands(rng, 120, 120, r, len(col_idx))
        dX0, stats0 = rng.standard_normal(X.shape), rng.standard_normal((120, 2))
        wdX, wstats, ws, _ = ref_bce(rowStart, col_idx, y, X, Y, 0.5, dX0, stats0)
        assert run_bce(rowStart, col_idx, y, X, Y, 0.5, scores=False) == (None, None, None)  # all null: a no-op
        d, st, sc = run_bce(rowStart, col_idx, y, X, Y, 0.5, dX0=dX0, scores=False)
        assert st is None and sc is None and np.abs(d - wdX).max() <= 1e-12 * np.abs(wdX).max()
        d, st, sc = run_bce(rowStart, col_idx, y, X, Y, 0.5, stats0=stats0, scores=False)
        assert d is None and np.abs(st[:, 0] - wstats[:, 0]).max() <= 1e-12 * np.abs(wstats[:, 0]).max()
        d, st, sc = run_bce(rowStart, col_idx, y, X, Y, 0.5)
        assert np.abs(sc - ws).max() <= 1e-12 * max(np.abs(ws).max(), 1.0)


@pytest.mark.parametrize("r,n", [(4, 200000), (64, 30000), (256, 12000), (5, 40000)])
def test_link_kernel_past_one_wave(world, r, n):
    rng = np.random.default_rng(SEED + n)
    rowStart, col_idx = csr_block(rng, n, 5000, per_row=3)
    X, Y, y = operands(rng, n, 5000, r, len(col_idx))
    check_bce(rowStart, col_idx, y, X, Y, inv=1.0 / len(col_idx))


@pytest.mark.parametrize("r", [64, 257])
def test_link_kernel_on_the_skewed_graph(world, r):
    rows, cols = skewed_tuples(4200, 4200, SEED)
    rows, cols = rows.astype(np.int64), cols.astype(np.int64)
    order = np.lexsort((cols, rows))
    rows, cols = rows[order], cols[order]
    rowStart = np.searchsorted(rows, np.arange(4201)).astype(np.int64)
    rng = np.random.default_rng(SEED + r)
    X, Y, y = operands(rng, 4200, 4200, r, len(cols))
    check_bce(rowStart, cols, y, X, Y, inv=1.0 / len(cols))
    # and its transpose (the B-order pass): the hub column becomes a hub row
    order = np.lexsort((rows, cols))
    tr, tc = cols[order], rows[order]
    check_bce(np.searchsorted(tr, np.arange(4201)).astype(np.int64), tc, y[order], Y, X, inv=1.0 / len(cols))


# ---- the distributed op at p = 1 ---------------------------------------------------------------------------------------
def targets(rng, N, n, dup=True, soft=True):
    tr, tc = rng.integers(0, N, n), rng.integers(0, N, n)
    if dup:
        tr[:9], tc[:9] = tr[9:18], tc[9:18]
    y = rng.choice([0.0, 1.0, 0.25] if soft else [0.0, 1.0], n)
    if dup:
        y[:9] = y[9:18]
    return tr.astype(np.int64), tc.astype(np.int64), y


def _dense(M):
    d = D.Dense.create(*M.shape)
    d.from_host(np.ascontiguousarray(M))
    return d


@pytest.mark.parametrize("name", ALGS)
def test_link_loss_op_at_p1(world, name):
    rng = np.random.default_rng(SEED + len(name))
    N, r = 300, 16
    tr, tc, y = targets(rng, N, 2000)
    tr[:50] = 7  # a hub row
    T = D.SpmatLocal.from_tuples(N, N, tr, tc, y)
    alg = D.Algorithm(name, T, r, 1)
    rows = alg.like_A_matrix().shape[0]
    assert rows == alg.like_B_matrix().shape[0]
    H = rng.standard_normal((rows, r)) / 2
    H[5] *= 40.0
    Hd, dHd = _dense(H), _dense(np.full((rows, r), math.nan))
    scores = alg.like_S_values()
    loss, correct, count = alg.link_loss(Hd, Hd, dHd, dHd, scores)
    wl, wc, wn, ws, wg, _ = lpo.link_loss(H[:N], H[:N], tr, tc, y, same=True)
    assert abs(loss - wl) <= 1e-12 * abs(wl) and count == wn == 2000
    assert abs(correct - wc) <= 2  # a score within rounding of 0 may count either way
    dH = dHd.to_host()
    assert np.abs(dH[:N] - wg).max() <= 1e-12 * np.abs(wg).max() and not dH[N:].any()
    er, ec = alg.entry_coordinates("A")
    key = {}
    for i, (u, v) in enumerate(zip(tr, tc)):
        key.setdefault((u, v), []).append(ws[i])
    got = scores.to_host()
    assert all(abs(s - key[(u, v)][0]) <= 1e-12 * max(abs(s), 1) for s, u, v in zip(got, er, ec))
    # separate H_A, H_B and gradients, and a forward-only call
    H2 = rng.standard_normal((rows, r))
    dA, dB = _dense(np.zeros((rows, r))), _dense(np.zeros((rows, r)))
    alg.link_loss(Hd, _dense(H2), dA, dB)
    _, _, _, _, gA, gB = lpo.link_loss(H[:N], H2[:N], tr, tc, y)
    assert np.abs(dA.to_host()[:N] - gA).max() <= 1e-12 * np.abs(gA).max()
    assert np.abs(dB.to_host()[:N] - gB).max() <= 1e-12 * np.abs(gB).max()
    l2 = alg.link_loss(Hd, Hd)
    assert l2 == (loss, correct, count)  # bit-identical, with or without gradients
    assert alg.link_loss(Hd, Hd, dHd, dHd, scores) == (loss, correct, count) and np.array_equal(dHd.to_host(), dH)


def test_link_refusals(world):
    rng = np.random.default_rng(SEED + 9)
    N, r = 128, 8
    rows, cols, _ = orc.er_tuples(7, 5, SEED)
    S = D.SpmatLocal.from_tuples(N, N, rows, cols, np.ones(len(rows)))
    alg = D.Algorithm("15d_fusion1", S, 6, 1)
    net = D.GraphTransformer(alg, [(6, 4, 2), (8, 8, 1)])
    tr, tc, y = targets(rng, N, 400)
    algT = D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, tr, tc, y), 6, 1)
    n = algT.like_A_matrix().shape[0]
    H, dH = _dense(rng.standard_normal((n, r))), _dense(np.zeros((n, r)))
    for args, what in (((_dense(np.zeros((n + 1, r))), H), "like_A_matrix"), ((H, _dense(np.zeros((n, r + 1)))), "one width"),
                       ((H, H, H), "may not be H_A"), ((H, H, None, H), "may not be H_A"),
                       ((H, H, _dense(np.zeros((n, r - 1)))), "dH_A is"), ((H, H, None, None, D.Vec.create(len(y) + 1)), "scores")):
        with pytest.raises(RuntimeError, match="link_loss failed") as e:
            algT.link_loss(*args)
        assert what in str(e.value), (what, str(e.value))
    # targets: another fusion, another size, values outside [0, 1]
    for alg_name, M_, vals in (("15d_fusion2", N, y), ("15d_fusion1", N + 1, y)):
        other = D.Algorithm(alg_name, D.SpmatLocal.from_tuples(M_, M_, tr, tc, vals), 6, 1)
        with pytest.raises(RuntimeError, match="layout"):
            D.LinkTargets(net, other)
    for bad in (1.5, -0.1, math.nan, math.inf):
        v = y.copy()
        v[17] = bad
        with pytest.raises(RuntimeError, match="not in \\[0, 1\\]"):
            D.LinkTargets(net, D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, tr, tc, v), 6, 1))
    t = D.LinkTargets(net, algT)
    assert t.alg_T is algT
    # an optimizer of other parameters, and targets of another model's algorithm object
    opt = D.AdamW(lr=1e-2)
    other_alg = D.Algorithm("15d_fusion1", S, 6, 1)
    other = D.GraphTransformer(other_alg, [(6, 2, 2), (4, 8, 1)])
    other.set_input(rng.standard_normal(other.buffer_shape(0)))
    other.link_train_step(D.LinkTargets(other, algT), opt)
    with pytest.raises(RuntimeError, match="parameters"):
        net.link_train_step(t, opt)
    with pytest.raises(RuntimeError, match="another model"):
        other.link_train_step(t, D.AdamW())
    with pytest.raises(RuntimeError, match="another model"):
        other.link_evaluate(t)


# ---- the models --------------------------------------------------------------------------------------------------------
def _graph(logM, npr, seed):
    rows, cols, _ = orc.er_tuples(logM, npr, seed)
    return np.asarray(rows, np.int64), np.asarray(cols, np.int64)


def check_steps(got, want):
    for t, (g, w) in enumerate(zip(got, want)):
        assert abs(g.loss - w[0]) <= 1e-10 * abs(w[0]), (t, g, w)
        assert (g.correct, g.labelled) == (w[1], w[2]), (t, g, w)
        assert abs(g.grad_norm - w[3]) <= 1e-10 * abs(w[3]), (t, g, w)


def _close(got, want, tol):
    return np.abs(got - want).max() <= tol * max(np.abs(want).max(), 1.0)


GT_CASES = {
    "plain": dict(layers=[(6, 4, 2), (8, 8, 1)], edge_dim=0, beta=False, ffn=0, dropout=0.0, clip=None, soft=False),
    "blocks_gate_edge": dict(layers=[(6, 4, 2), (8, 3, 2)], edge_dim=3, beta=True, ffn=2, dropout=0.0, clip=None, soft=True),
    "dropout_clip_schedule": dict(layers=[(6, 4, 2), (8, 5, 1)], edge_dim=2, beta=True, ffn=1, dropout=0.3, clip=0.05, soft=True),
}


def _gt_setup(name, rng, alg, net, N):
    cfg = GT_CASES[name]
    params = gbo.random_params(cfg["layers"], cfg["edge_dim"], cfg["beta"], cfg["ffn"], rng)
    for l, P in enumerate(params):
        for k, v in P.items():
            net.set_param(l, k, v)
    X = rng.uniform(-1, 1, (N, cfg["layers"][0][0]))
    net.set_input(np.vstack([X, np.zeros((net.buffer_shape(0)[0] - N, X.shape[1]))]))
    if cfg["edge_dim"]:
        net.set_edge_attributes(attr_of(*alg.entry_coordinates("A"), cfg["edge_dim"]),
                                attr_of(*alg.entry_coordinates("B"), cfg["edge_dim"]))
    return params, X


@pytest.mark.parametrize("name", sorted(GT_CASES))
def test_graph_transformer_link_train_steps_match_torch(world, name):
    cfg, steps, N = GT_CASES[name], 5, 128
    layers = cfg["layers"]
    rows, cols = _graph(7, 5, SEED)
    S = D.SpmatLocal.from_tuples(N, N, rows, cols, np.ones(len(rows)))
    alg = D.Algorithm("15d_fusion1", S, layers[0][0], 1)
    net = D.GraphTransformer(alg, layers, edge_dim=cfg["edge_dim"], beta=cfg["beta"], ffn_ratio=cfg["ffn"])
    rng = np.random.default_rng(SEED + len(name))
    params, X = _gt_setup(name, rng, alg, net, N)
    tr, tc, y = targets(rng, N, 600, soft=cfg["soft"])
    algT = D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, tr, tc, y), layers[0][0], 1)
    t = D.LinkTargets(net, algT)
    lrs = [1e-2, 2e-2, 3e-2, 2e-2, 1e-2] if cfg["clip"] else [1e-2] * steps
    opt = D.AdamW(lr=lrs[0], weight_decay=0.01, max_grad_norm=cfg["clip"])
    seeds = [11 + 7 * s for s in range(steps)]
    got = []
    for s in range(steps):
        opt.lr = lrs[s]
        got.append(net.link_train_step(t, opt, cfg["dropout"], seeds[s]))
    want, tparams = lpo.train_gt(rows, cols, N, layers, params, X, (tr, tc, y), steps,
                                 attr=attr_of(rows, cols, cfg["edge_dim"]) if cfg["edge_dim"] else None, beta=cfg["beta"],
                                 ffn=cfg["ffn"], dropout=cfg["dropout"], seeds=seeds, lr=lrs[0], lrs=lrs, weight_decay=0.01,
                                 max_grad_norm=cfg["clip"])
    check_steps(got, want)
    if cfg["clip"]:
        assert any(w[3] > cfg["clip"] for w in want)  # clipping was active
    for l, P in enumerate(tparams):
        for k, w in P.items():
            g = net.param(l, k)
            if k == "key_bias":  # its gradient is rounding noise on both sides; Adam turns it into steps of up to lr
                assert np.abs(g - w).max() <= sum(lrs) * 1.01, (l, k)
            else:
                assert _close(g, w, 1e-9), (name, l, k, np.abs(g - w).max())
    # link_evaluate: a forward without dropout and the scores in T's A order
    loss, correct, count, scores = net.link_evaluate(t)
    H = net.buffer(len(layers))[:N]
    wl, wc, wn, ws, _, _ = lpo.link_loss(H, H, tr, tc, y, same=True)
    assert abs(loss - wl) <= 1e-12 * abs(wl) and count == wn and abs(correct - wc) <= 1
    er, ec = algT.entry_coordinates("A")
    assert np.abs(scores - (H[er] * H[ec]).sum(1)).max() <= 1e-12 * max(np.abs(scores).max(), 1.0)


@pytest.mark.parametrize("kind", ["leaky", "softmax", "additive", "gatv2"])
def test_gat_link_train_steps_match_torch(world, kind):
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
    tr, tc, y = targets(rng, N, 500)
    t = D.LinkTargets(net, D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, tr, tc, y), layers[0][0], 1))
    opt = D.AdamW(lr=1e-2)
    got = [net.link_train_step(t, opt) for _ in range(steps)]
    want, ws, u1, u2 = lpo.train_gat(kind, rows, cols, N, layers, weights, a1, a2, X, (tr, tc, y), steps, lr=1e-2)
    check_steps(got, want)
    for l, (f, d, H) in enumerate(layers):
        for h in range(H):
            assert _close(net.weight(l, h), ws[l][h], 1e-9), (kind, l, h)
            v1, v2 = net.attention_vectors(l, h)
            assert _close(v1, u1[l][h], 1e-9) and _close(v2, u2[l][h], 1e-9), (kind, l, h)
    _, _, _, scores = net.link_evaluate(t)
    assert (scores >= 0).all()  # the last layer's ReLU


# ---- convergence -------------------------------------------------------------------------------------------------------
def test_graph_transformer_learns_links_of_a_block_model(world):
    """A stochastic block model of 4 blocks: S holds 80 % of the intra-block edges and a few cross-block ones; the model
    trains on S's edges against as many random cross-block pairs, and is evaluated on the held-out intra-block edges
    against fresh cross-block pairs.  100 steps halve the loss and the held-out AUC reaches 0.85."""
    N, B, f = 256, 4, 8
    rng = np.random.default_rng(SEED + 7)
    block = np.arange(N) * B // N
    same = block[:, None] == block[None, :]
    intra = np.argwhere(same & (rng.random((N, N)) < 0.12) & ~np.eye(N, dtype=bool))
    rng.shuffle(intra)
    cut = int(0.8 * len(intra))
    train_e, held = intra[:cut], intra[cut:]
    cross = np.argwhere(~same & (rng.random((N, N)) < 0.004))
    edges = np.vstack([train_e, cross])
    S = D.SpmatLocal.from_tuples(N, N, edges[:, 0], edges[:, 1], np.ones(len(edges)))
    alg = D.Algorithm("15d_fusion1", S, f, 1)

    def negatives(n):
        u, v = rng.integers(0, N, 4 * n), rng.integers(0, N, 4 * n)
        keep = block[u] != block[v]
        return u[keep][:n], v[keep][:n]

    def target_alg(pos):
        nu, nv = negatives(len(pos))
        tr, tc = np.concatenate([pos[:, 0], nu]), np.concatenate([pos[:, 1], nv])
        y = np.concatenate([np.ones(len(pos)), np.zeros(len(nu))])
        return D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, tr, tc, y), f, 1), y

    train_alg, _ = target_alg(train_e)
    test_alg, _ = target_alg(held)
    net = D.GraphTransformer(alg, [(f, 8, 2), (16, 8, 1)])
    for l, P in enumerate(gbo.random_params([(f, 8, 2), (16, 8, 1)], 0, False, 0, rng, scale=0.3)):
        for k, v in P.items():
            net.set_param(l, k, v)
    X = 0.5 * rng.standard_normal((N, f))
    X[np.arange(N), block] += 1.0  # noisy block indicators
    net.set_input(np.vstack([X, np.zeros((net.buffer_shape(0)[0] - N, f))]))
    t_train, t_test = D.LinkTargets(net, train_alg), D.LinkTargets(net, test_alg)
    opt = D.AdamW(lr=2e-2, weight_decay=0.0)
    hist = [net.link_train_step(t_train, opt) for _ in range(100)]
    assert hist[-1].loss < 0.5 * hist[0].loss, (hist[0], hist[-1])
    loss, correct, count, scores = net.link_evaluate(t_test)
    er, ec = test_alg.entry_coordinates("A")
    y = (block[er] == block[ec]).astype(float)  # held-out positives are intra-block, negatives cross-block
    assert lpo.auc(scores, y) >= 0.85, (lpo.auc(scores, y), loss, correct, count)
