"""Relation-aware link prediction on the GPU on one rank.  The kernels hnh_distmult_bce_f64 / _grad_f64 against numpy at
the table widths and odd ones from r = 1 to 257, odd leading dimensions and misaligned rows, rows without entries,
duplicates, values that are no relation, past one resident wave and on the skewed graph (tests/skewed_graph.py), with
bit-identical repeats, and R = 1 with D = 1 against hnh_link_bce_f64.  The op Distributed_Sparse::distmultLoss at p = 1
under every algorithm name against tests/distmult_oracle.py, its dD at the table widths and odd ones, accumulation of a
positive and a negative call, duplicate pairs under different relations, an empty T and bit-identical repeats of every
output.  Relational link train steps of R-GCN (plain and with bases) and of the graph transformer against a torch AdamW
loop, evaluate's scores, every refusal, and a learning check that dot-product link prediction cannot pass.  Multi-rank
cases are in tests/test_distmult_multirank_gpu.py."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from distributed_sddmm_b200 import driver as D
from distributed_sddmm_b200 import lib
from oracle import hnh_oracle as orc
from tests import distmult_oracle as dmo
from tests import graph_transformer_block_oracle as gbo
from tests import graph_transformer_oracle as gto
from tests import rgcn_basis_oracle as bo
from tests import rgcn_oracle as ro
from tests.skewed_graph import skewed_tuples
from tests.test_link_prediction_gpu import _dev_rows, csr_block

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
SEED = 0xC0FFEE + 409
ALGS = ["15d_fusion1", "15d_fusion2", "15d_sparse", "25d_dense_replicate", "25d_sparse_replicate"]


@pytest.fixture(scope="module")
def world():
    D.world_init("self")
    yield
    D.world_finalize()


def _st():
    return torch.cuda.current_stream().cuda_stream


# ---- the kernels ----------------------------------------------------------------------------------------------------------
def run_bce(rowStart, col_idx, rels, R, X, Y, Dt, target, inv, dX0, stats0=None, grad=False, ld=None, offset=0, outs=True):
    """Runs hnh_distmult_bce_f64 (grad: _grad_f64); returns (dX, stats, scores, g) as numpy (None where not asked)."""
    n, r = X.shape
    ldx, ldy, ldd, lddx = ld or (r, r, r, r)
    xb, yb, db = _dev_rows(X, ldx, offset), _dev_rows(Y, ldy, offset), _dev_rows(Dt, ldd, offset)
    rs, ci = torch.from_numpy(rowStart).to(DEV), torch.from_numpy(col_idx).to(DEV)
    rv = torch.from_numpy(np.asarray(rels, np.float64)).to(DEV)
    gx = _dev_rows(dX0, lddx, offset)
    p = lambda b, off=0: b.data_ptr() + 8 * off if b is not None else None  # noqa: E731
    if grad:
        rc = lib().hnh_distmult_bce_grad_f64(rs.data_ptr(), ci.data_ptr(), rv.data_ptr(), n, len(col_idx), R, p(xb, offset), ldx,
                                             p(yb, offset), ldy, p(db, offset), ldd, r, target, inv, p(gx, offset), lddx, _st())
        sb = sc = gv = None
    else:
        sb = torch.from_numpy(stats0.copy()).to(DEV)
        sc = torch.full((len(col_idx) + 1,), math.nan, dtype=torch.float64, device=DEV) if outs else None
        gv = torch.full((len(col_idx) + 1,), math.nan, dtype=torch.float64, device=DEV) if outs else None
        rc = lib().hnh_distmult_bce_f64(rs.data_ptr(), ci.data_ptr(), rv.data_ptr(), n, len(col_idx), R, p(xb, offset), ldx,
                                        p(yb, offset), ldy, p(db, offset), ldd, r, target, inv, p(gx, offset), lddx, p(sb), 2,
                                        p(sc), p(gv), _st())
    assert rc == 0, lib().hnh_last_error_string()
    torch.cuda.synchronize()
    d = gx[offset:offset + n * lddx].view(n, lddx)
    if lddx > r:
        assert torch.isnan(d[:, r:]).all()  # the columns past r are not written
    h = lambda b: b[:-1].cpu().numpy() if b is not None else None  # noqa: E731
    if sc is not None:
        assert torch.isnan(sc[-1]) and torch.isnan(gv[-1])
    return d[:, :r].cpu().numpy(), sb.cpu().numpy() if sb is not None else None, h(sc), h(gv)


def ref_bce(rowStart, col_idx, rels, R, X, Y, Dt, target, inv, dX0, stats0):
    rows = np.repeat(np.arange(len(rowStart) - 1), np.diff(rowStart))
    ok = ro.valid(rels, R)
    rho = np.where(ok, np.nan_to_num(np.asarray(rels, np.float64)), 0).astype(np.int64)
    s = np.where(ok, (X[rows] * Dt[rho] * Y[col_idx]).sum(1), 0.0)
    st = torch.from_numpy(s)
    loss = np.where(ok, F.binary_cross_entropy_with_logits(st, torch.full_like(st, target), reduction="none").numpy(), 0.0)
    g = np.where(ok, (torch.sigmoid(st).numpy() - target) * inv, 0.0)
    dX = dX0.copy()
    np.add.at(dX, rows, g[:, None] * Dt[rho] * Y[col_idx])
    stats = stats0.copy()
    np.add.at(stats[:, 0], rows, loss)
    np.add.at(stats[:, 1], rows, (ok & ((s > 0) == (target > 0.5))).astype(np.float64))
    bound = (np.abs(X[rows]) * np.abs(Dt[rho]) * np.abs(Y[col_idx])).sum(1)
    return dX, stats, s, g, bound


def operands(rng, n, m, r, R, nnz, bad=True):
    X = rng.standard_normal((n, r)) / r ** 0.25
    Y = rng.standard_normal((m, r)) / r ** 0.25
    Dt = rng.uniform(0.5, 2.0, (R, r)) * rng.choice([-1.0, 1.0], (R, r))
    X[rng.random(n) < 0.1] *= 100.0
    rels = rng.integers(0, R, nnz).astype(np.float64)
    if bad and nnz > 8:
        rels[rng.choice(nnz, 5, replace=False)] = [-1.0, float(R), 0.5, math.nan, math.inf]  # no relation
    return X, Y, Dt, rels


def check_bce(rowStart, col_idx, rels, R, X, Y, Dt, target=1.0, inv=1e-2, **kw):
    rng = np.random.default_rng(len(col_idx))
    dX0, stats0 = rng.standard_normal(X.shape), rng.standard_normal((X.shape[0], 2))
    stats0[:, 1] = rng.integers(0, 5, len(stats0))
    got = run_bce(rowStart, col_idx, rels, R, X, Y, Dt, target, inv, dX0, stats0, **kw)
    dX, stats, s, g = got
    wdX, wstats, ws, wg, bound = ref_bce(rowStart, col_idx, rels, R, X, Y, Dt, target, inv, dX0, stats0)
    assert (np.abs(s - ws) <= 1e-13 * bound + 1e-300).all()
    assert np.abs(dX - wdX).max() <= 1e-12 * max(np.abs(wdX).max(), 1.0)
    assert np.abs(g - wg).max() <= 1e-12 * max(np.abs(wg).max(), 1e-300)
    assert np.abs(stats[:, 0] - wstats[:, 0]).max() <= 1e-12 * max(np.abs(wstats[:, 0]).max(), 1.0)
    rows = np.repeat(np.arange(len(rowStart) - 1), np.diff(rowStart))
    near0 = np.zeros(len(stats), bool)
    np.logical_or.at(near0, rows, np.abs(ws) <= 1e-12 * bound)
    assert np.array_equal(stats[~near0, 1], wstats[~near0, 1])
    empty = np.diff(rowStart) == 0
    assert np.array_equal(dX[empty], dX0[empty]) and np.array_equal(stats[empty], stats0[empty])
    again = run_bce(rowStart, col_idx, rels, R, X, Y, Dt, target, inv, dX0, stats0, **kw)
    assert all(np.array_equal(a, b) for a, b in zip(got, again))  # bit-identical repeats
    # the B-order kernel gives the same dX
    gdX, *_ = run_bce(rowStart, col_idx, rels, R, X, Y, Dt, target, inv, dX0, grad=True, **kw)
    assert np.abs(gdX - wdX).max() <= 1e-12 * max(np.abs(wdX).max(), 1.0)


WIDTHS = [1, 3, 4, 8, 16, 32, 33, 64, 128, 256, 257]


@pytest.mark.parametrize("r", WIDTHS)
def test_distmult_kernel_matches_numpy(world, r):
    rng = np.random.default_rng(SEED + r)
    rowStart, col_idx = csr_block(rng, 300, 400)
    X, Y, Dt, rels = operands(rng, 300, 400, r, 5, len(col_idx))
    for target in (1.0, 0.0):
        check_bce(rowStart, col_idx, rels, 5, X, Y, Dt, target=target)


@pytest.mark.parametrize("r", [3, 4, 64, 256, 257])
def test_distmult_kernel_odd_ld_and_misaligned(world, r):
    rng = np.random.default_rng(SEED + 2 * r)
    rowStart, col_idx = csr_block(rng, 200, 150)
    X, Y, Dt, rels = operands(rng, 200, 150, r, 3, len(col_idx))
    for ld, offset in (((r + 1, r, r, r), 0), ((r, r + 1, r, r), 0), ((r, r, r + 1, r), 0), ((r, r, r, r + 1), 0),
                       ((r, r, r, r), 1), ((r + 3, r + 2, r + 1, r + 1), 1)):
        check_bce(rowStart, col_idx, rels, 3, X, Y, Dt, ld=ld, offset=offset)


@pytest.mark.parametrize("r,n", [(4, 200000), (64, 30000), (256, 12000), (5, 40000)])
def test_distmult_kernel_past_one_wave(world, r, n):
    rng = np.random.default_rng(SEED + n)
    rowStart, col_idx = csr_block(rng, n, 5000, per_row=3)
    X, Y, Dt, rels = operands(rng, n, 5000, r, 7, len(col_idx))
    check_bce(rowStart, col_idx, rels, 7, X, Y, Dt, inv=1.0 / len(col_idx))


@pytest.mark.parametrize("r", [64, 257])
def test_distmult_kernel_on_the_skewed_graph(world, r):
    rows, cols = skewed_tuples(4200, 4200, SEED)
    rows, cols = rows.astype(np.int64), cols.astype(np.int64)
    order = np.lexsort((cols, rows))
    rows, cols = rows[order], cols[order]
    rng = np.random.default_rng(SEED + r)
    X, Y, Dt, rels = operands(rng, 4200, 4200, r, 4, len(cols))
    check_bce(np.searchsorted(rows, np.arange(4201)).astype(np.int64), cols, rels, 4, X, Y, Dt, inv=1.0 / len(cols))


def test_distmult_kernel_r1_d1_is_link_bce(world):
    """R = 1 with D = 1 gives the dot-product decoder: hnh_link_bce_f64's bits, within 1e-12 in any case."""
    rng = np.random.default_rng(SEED + 3)
    rowStart, col_idx = csr_block(rng, 500, 500)
    for r in (64, 7):
        X, Y, _, _ = operands(rng, 500, 500, r, 1, len(col_idx))
        dX0, stats0 = np.zeros(X.shape), np.zeros((500, 2))
        dX, stats, s, _ = run_bce(rowStart, col_idx, np.zeros(len(col_idx)), 1, X, Y, np.ones((1, r)), 1.0, 0.01, dX0, stats0)
        from tests.test_link_prediction_gpu import run_bce as link_bce
        ldX, lstats, ls = link_bce(rowStart, col_idx, np.ones(len(col_idx)), X, Y, 0.01, dX0, stats0)
        assert np.abs(s - ls).max() <= 1e-12 * np.abs(ls).max()
        assert np.abs(dX - ldX).max() <= 1e-12 * np.abs(ldX).max()
        assert np.abs(stats - lstats).max() <= 1e-12 * np.abs(lstats).max()


# ---- the distributed op at p = 1 ---------------------------------------------------------------------------------------
def _dense(M):
    d = D.Dense.create(*M.shape)
    d.from_host(np.ascontiguousarray(M))
    return d


def triples(rng, N, R, n):
    tr, tc, rels = rng.integers(0, N, n), rng.integers(0, N, n), rng.integers(0, R, n).astype(np.float64)
    tr[:9], tc[:9] = tr[9:18], tc[9:18]  # the same pairs, under their own relations
    rels[:9] = (rels[9:18] + 1) % R
    tr[20:70] = 7  # a hub row
    return tr.astype(np.int64), tc.astype(np.int64), rels


def _close(got, want, tol=1e-12):
    return np.abs(got - want).max() <= tol * max(np.abs(want).max(), 1e-300)


def run_op(alg, H, H2, Dt, R, target, inv, accumulate=False, dHs=None, dD=None, scores=True):
    Hd = _dense(H)
    H2d = Hd if H2 is None else _dense(H2)
    dA = dHs[0] if dHs else _dense(np.zeros(H.shape))
    dB = dHs[1] if dHs else (dA if H2 is None else _dense(np.zeros(H.shape)))
    dDd = dD if dD is not None else _dense(np.zeros(Dt.shape))
    sc = alg.like_S_values() if scores else None
    res = alg.distmult_loss(Hd, H2d, _dense(Dt), R, target, inv, dA, dB, dDd, sc, accumulate=accumulate)
    return res, dA, dB, dDd, sc


def check_scores(alg_T, got, trip, want):
    """got (A order) against want (in the order of trip = (rows, cols, rels)) as multisets per (u, v): a pair stored
    under several relations has one score per relation."""
    er, ec = alg_T.entry_coordinates("A")
    g, w = {}, {}
    for s, u, v in zip(got, er, ec):
        g.setdefault((u, v), []).append(s)
    for s, u, v in zip(want, trip[0], trip[1]):
        w.setdefault((u, v), []).append(s)
    assert g.keys() == w.keys()
    scale = max(np.abs(want).max(), 1.0)
    for k in g:
        assert np.abs(np.sort(g[k]) - np.sort(w[k])).max() <= 1e-12 * scale, k


@pytest.mark.parametrize("name", ALGS)
def test_distmult_op_at_p1(world, name):
    rng = np.random.default_rng(SEED + len(name))
    N, r, R = 300, 16, 6
    tr, tc, rels = triples(rng, N, R, 2000)
    alg = D.Algorithm(name, D.SpmatLocal.from_tuples(N, N, tr, tc, rels), r, 1)
    rows = alg.like_A_matrix().shape[0]
    H = rng.standard_normal((rows, r)) / 2
    H[5] *= 20.0
    Dt = rng.standard_normal((R, r))
    inv = 1.0 / 4000
    (ls, c), dA, _, dD, sc = run_op(alg, H, None, Dt, R, 1.0, inv)
    wl, wc, ws, wg, _, wd = dmo.op(H[:N], H[:N], Dt, tr, tc, rels, 1.0, inv, same=True)
    assert abs(ls - wl) <= 1e-12 * wl and abs(c - wc) <= 2
    assert _close(dA.to_host()[:N], wg) and not dA.to_host()[N:].any() and _close(dD.to_host(), wd)
    check_scores(alg, sc.to_host(), (tr, tc, rels), ws)
    assert len({round(w, 9) for w in ws[:18]}) == 18  # the duplicated pairs score once per relation
    # a negative call accumulated onto the positive one: the gradients of the mean over both
    dN = run_op(alg, H, None, Dt, R, 0.0, inv, accumulate=True, dHs=(dA, dA), dD=dD)
    nl, nc, _, ng, _, nd = dmo.op(H[:N], H[:N], Dt, tr, tc, rels, 0.0, inv, same=True)
    assert abs(dN[0][0] - nl) <= 1e-12 * nl
    assert _close(dA.to_host()[:N], wg + ng) and _close(dD.to_host(), wd + nd)
    # separate H_A, H_B and gradients
    H2 = rng.standard_normal((rows, r))
    _, dA2, dB2, dD2, _ = run_op(alg, H, H2, Dt, R, 1.0, inv)
    _, _, _, gA, gB, gD = dmo.op(H[:N], H2[:N], Dt, tr, tc, rels, 1.0, inv)
    assert _close(dA2.to_host()[:N], gA) and _close(dB2.to_host()[:N], gB) and _close(dD2.to_host(), gD)
    # bit-identical repeats of every output
    first = run_op(alg, H, None, Dt, R, 1.0, inv)
    again = run_op(alg, H, None, Dt, R, 1.0, inv)
    assert first[0] == again[0] == (ls, c)
    for a, b in zip(first[1:], again[1:]):
        assert np.array_equal(a.to_host(), b.to_host())


@pytest.mark.parametrize("r", [1, 3, 4, 8, 33, 64, 128, 256, 257])
def test_distmult_relation_gradient_widths(world, r):
    rng = np.random.default_rng(SEED + 5 * r)
    N, R = 400, 237
    tr, tc, rels = triples(rng, N, R, 6000)
    rels[:1500] = 3  # one relation of more than one piece
    bad = rels.copy()
    bad[100:105] = [-1.0, float(R), 0.5, math.nan, math.inf]
    alg = D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, tr, tc, bad), r, 1)
    H = rng.standard_normal((alg.like_A_matrix().shape[0], r))
    Dt = rng.standard_normal((R, r))
    (ls, c), dA, _, dD, sc = run_op(alg, H, None, Dt, R, 1.0, 1e-3)
    wl, wc, _, wg, _, wd = dmo.op(H[:N], H[:N], Dt, tr, tc, bad, 1.0, 1e-3, same=True)
    assert abs(ls - wl) <= 1e-12 * wl and _close(dA.to_host()[:N], wg) and _close(dD.to_host(), wd)
    again = run_op(alg, H, None, Dt, R, 1.0, 1e-3)
    assert np.array_equal(again[3].to_host(), dD.to_host())


def test_distmult_op_empty_and_sums(world):
    rng = np.random.default_rng(SEED + 6)
    N, r, R = 64, 8, 3
    alg = D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, [], [], []), r, 1)
    H = rng.standard_normal((alg.like_A_matrix().shape[0], r))
    res, dA, _, dD, sc = run_op(alg, H, None, rng.standard_normal((R, r)), R, 1.0, 0.0)
    assert res == (0.0, 0) and not dA.to_host().any() and not dD.to_host().any() and len(sc) == 0


def test_distmult_op_refusals(world):
    rng = np.random.default_rng(SEED + 7)
    N, r, R = 128, 8, 3
    tr, tc, rels = triples(rng, N, R, 400)
    alg = D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, tr, tc, rels), r, 1)
    n = alg.like_A_matrix().shape[0]
    H, Dt = _dense(rng.standard_normal((n, r))), _dense(rng.standard_normal((R, r)))
    z = lambda *s: _dense(np.zeros(s))  # noqa: E731
    for args, kw, what in (((H, H, z(R + 1, r), R), {}, "D is"), ((H, H, z(R, r + 1), R), {}, "like_A_matrix|D is"),
                           ((H, H, Dt, 0), {}, "relation count"), ((H, H, Dt, R), dict(target=1.5), "target"),
                           ((H, H, Dt, R), dict(inv_count=-1.0), "inv_count"), ((H, H, Dt, R), dict(dD=z(R, r - 1)), "dD is"),
                           ((H, H, Dt, R), dict(dD=Dt), "may not be"), ((H, H, Dt, R), dict(dH_A=H), "may not be"),
                           ((H, H, Dt, R), dict(scores=D.Vec.create(3)), "scores")):
        k = dict(target=1.0, inv_count=0.1)
        k.update(kw)
        with pytest.raises(RuntimeError, match="distmult_loss failed") as e:
            alg.distmult_loss(*args, **k)
        assert any(w in str(e.value) for w in what.split("|")), (what, str(e.value))


# ---- models ------------------------------------------------------------------------------------------------------------
def _rgcn(layers, R, B, seed, aggr="mean"):
    N = 128
    rows, cols, _ = orc.er_tuples(7, 5, seed)
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    rels = np.random.default_rng(seed + 2).integers(0, R, len(rows)).astype(np.float64)
    alg = D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, rows, cols, rels), layers[0][0], 1)
    net = D.RGCN(alg, layers, num_relations=R, aggr=aggr, num_bases=B)
    rng = np.random.default_rng(seed + 1)
    params = bo.random_params(layers, R, B, rng) if B else ro.random_params(layers, R, rng)
    for l, P in enumerate(params):
        for k, v in P.items():
            net.set_param(l, k, v)
    X = rng.uniform(-1, 1, (N, layers[0][0]))
    net.set_input(np.vstack([X, np.zeros((net.buffer_shape(0)[0] - N, X.shape[1]))]))
    if B:
        fwd = lambda tp, x: bo.model_torch(rows, cols, rels, N, layers, tp, x, R, B, aggr)  # noqa: E731
    else:
        fwd = lambda tp, x: ro.model_torch(rows, cols, rels, N, layers, tp, x, R, aggr)  # noqa: E731
    return dict(N=N, alg=alg, net=net, params=params, X=X, fwd=fwd)


def _gt(layers, seed):
    N = 128
    rows, cols, _ = orc.er_tuples(7, 5, seed)
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    alg = D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, rows, cols, np.ones(len(rows))), layers[0][0], 1)
    net = D.GraphTransformer(alg, layers)
    rng = np.random.default_rng(seed + 1)
    params = gbo.random_params(layers, 0, False, 0, rng)
    for l, P in enumerate(params):
        for k, v in P.items():
            net.set_param(l, k, v)
    X = rng.uniform(-1, 1, (N, layers[0][0]))
    net.set_input(np.vstack([X, np.zeros((net.buffer_shape(0)[0] - N, X.shape[1]))]))
    fwd = lambda tp, x: gto.model_torch(rows, cols, N, layers, tp, x)  # noqa: E731
    return dict(N=N, alg=alg, net=net, params=params, X=X, fwd=fwd)


MODELS = {
    "rgcn": lambda: _rgcn([(6, 8), (8, 8)], 3, None, SEED + 20),
    "rgcn_bases": lambda: _rgcn([(6, 8), (8, 8)], 3, 2, SEED + 21, aggr="sum"),
    "graph_transformer": lambda: _gt([(6, 4, 2), (8, 8, 1)], SEED + 22),
}


def _targets_algs(rng, N, R, n_pos, n_neg, f0):
    pos, neg = triples(rng, N, R, n_pos), triples(rng, N, R, n_neg)
    mk = lambda t: D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, *t), f0, 1)  # noqa: E731
    return pos, neg, mk(pos), mk(neg)


@pytest.mark.parametrize("model", sorted(MODELS))
def test_relational_link_train_steps_match_torch(world, model):
    P = MODELS[model]()
    net, N, R = P["net"], P["N"], 5
    rng = np.random.default_rng(SEED + len(model))
    pos, neg, alg_pos, alg_neg = _targets_algs(rng, N, R, 500, 400, P["X"].shape[1])
    dec = D.DistMultDecoder(net, R)
    assert dec.param_shape("rel") == (R, 8) and not dec.param("rel").any()
    torch.manual_seed(3)
    rel_emb = dmo.DistMultDecoder(R, 8).rel_emb.detach().numpy()  # a loaded state dict: rel_emb -> "rel"
    dec.set_param("rel", rel_emb)
    t = D.RelationalLinkTargets(net, alg_pos, alg_neg, R)
    opt = D.AdamW(lr=1e-2, max_grad_norm=1.0)
    got = [net.relational_link_train_step(dec, t, opt) for _ in range(4)]
    tp = [{k: dmo._t(v).clone().requires_grad_() for k, v in Pp.items()} for Pp in P["params"]]
    x = dmo._t(P["X"])
    want, rel = dmo.train(lambda _: P["fwd"](tp, x), [v for Pp in tp for v in Pp.values()], rel_emb, pos, neg, 4, lr=1e-2,
                          max_grad_norm=1.0)
    for g, w in zip(got, want):
        assert abs(g.loss - w[0]) <= 1e-10 * abs(w[0]) and abs(g.grad_norm - w[3]) <= 1e-10 * abs(w[3]), (g, w)
        assert g.labelled == w[2] == 900 and abs(g.correct - w[1]) <= 1
    assert _close(dec.param("rel"), rel, 1e-9)
    for l, Pp in enumerate(tp):
        for k, v in Pp.items():
            assert _close(net.param(l, k), v.detach().numpy(), 1e-9), (model, l, k)
    assert dec.param_grad("rel").shape == (R, 8)
    # evaluate: the scores in each matrix's A order
    loss, correct, count, sp, sn = net.relational_link_evaluate(dec, t)
    H, rel = net.buffer(len(net.layers))[:N], dec.param("rel")
    Ht, relt = torch.as_tensor(H), torch.as_tensor(rel)
    for alg_T, s, trip in ((alg_pos, sp, pos), (alg_neg, sn, neg)):
        check_scores(alg_T, s, trip, dmo.scores(Ht, Ht, relt, *trip)[0].numpy())
    wl, wc, wn, _, _ = dmo.relational_loss(torch.as_tensor(H), torch.as_tensor(rel), pos, neg)
    assert abs(loss - float(wl)) <= 1e-12 * float(wl) and count == wn == 900 and abs(correct - wc) <= 1


def test_relational_refusals(world):
    P = MODELS["rgcn"]()
    net, N, R = P["net"], P["N"], 3
    rng = np.random.default_rng(SEED + 30)
    pos, neg, alg_pos, alg_neg = _targets_algs(rng, N, R, 200, 100, 6)
    dec, t = D.DistMultDecoder(net, R), D.RelationalLinkTargets(net, alg_pos, alg_neg, R)
    # a relation out of range, or not an integer, in either matrix, and another layout
    for bad in (3.0, -1.0, 0.5, math.nan):
        rels = pos[2].copy()
        rels[17] = bad
        a = D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, pos[0], pos[1], rels), 6, 1)
        with pytest.raises(RuntimeError, match="not integers in"):
            D.RelationalLinkTargets(net, alg_pos, a, R)
    with pytest.raises(RuntimeError, match="layout"):
        D.RelationalLinkTargets(net, alg_pos, D.Algorithm("15d_fusion2", D.SpmatLocal.from_tuples(N, N, *neg), 6, 1), R)
    with pytest.raises(RuntimeError, match="relation count"):
        D.RelationalLinkTargets(net, alg_pos, alg_neg, 0)
    # a decoder of another R, another width (another model), targets and a decoder of another model's algorithm object
    other = MODELS["rgcn"]()
    for d_, t_, what in ((D.DistMultDecoder(net, R + 1), t, "relations"), (dec, D.RelationalLinkTargets(other["net"], *_targets_algs(
            rng, N, R, 50, 50, 6)[2:], R), "targets were made for another"), (D.DistMultDecoder(other["net"], R), t, "decoder was made")):
        with pytest.raises(RuntimeError, match=what):
            net.relational_link_train_step(d_, t_, D.AdamW())
        with pytest.raises(RuntimeError, match=what):
            net.relational_link_evaluate(d_, t_)
    narrow = D.RGCN(net.alg, [(6, 5)], num_relations=R)  # the same algorithm object, an output 5 wide
    with pytest.raises(RuntimeError, match="wide"):
        net.relational_link_train_step(D.DistMultDecoder(narrow, R), t, D.AdamW())
    # an optimizer of other parameters
    opt = D.AdamW()
    other["net"].link_train_step(D.LinkTargets(other["net"], D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(
        N, N, pos[0], pos[1], np.ones(len(pos[0]))), 6, 1)), opt)
    with pytest.raises(RuntimeError, match="parameters"):
        net.relational_link_train_step(dec, t, opt)
    with pytest.raises(RuntimeError, match="no relational train step"):
        dec.param_grad("rel")
    with pytest.raises(RuntimeError, match="no parameter"):
        dec.param_shape("weight")


# ---- learning ----------------------------------------------------------------------------------------------------------
def test_rgcn_with_distmult_learns_what_dot_products_cannot(world):
    """Every pair (u, v) of a set is a positive under one relation and a negative under the other: relation 0 holds
    the pairs of one community, relation 1 the pairs across communities.  A dot-product decoder scores a pair the same
    whatever its label, so it cannot exceed 0.5 accuracy; R-GCN with DistMult reaches 0.9 within 150 steps."""
    N, R, f = 128, 2, 8
    rng = np.random.default_rng(SEED + 40)
    comm = np.arange(N) % 2
    rows, cols, _ = orc.er_tuples(7, 6, SEED + 41)
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    srels = (comm[rows] != comm[cols]).astype(np.float64)  # the graph's own edges carry the same relation types
    alg = D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, rows, cols, srels), f, 1)
    net = D.RGCN(alg, [(f, 16), (16, 16)], num_relations=R, aggr="mean")
    for l, Pp in enumerate(ro.random_params([(f, 16), (16, 16)], R, rng, scale=0.5)):
        for k, v in Pp.items():
            net.set_param(l, k, v)
    X = rng.standard_normal((N, f))
    net.set_input(np.vstack([X, np.zeros((net.buffer_shape(0)[0] - N, f))]))
    u, v = rng.integers(0, N, 1500), rng.integers(0, N, 1500)
    same = (comm[u] == comm[v]).astype(np.float64)
    pos_rel, neg_rel = 1.0 - same, same  # the true relation, and the other one
    mk = lambda rr: D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, u, v, rr), f, 1)  # noqa: E731
    a_pos, a_neg = mk(pos_rel), mk(neg_rel)
    dec = D.DistMultDecoder(net, R)
    dec.set_param("rel", rng.uniform(-0.5, 0.5, (R, 16)))
    t = D.RelationalLinkTargets(net, a_pos, a_neg, R)
    opt = D.AdamW(lr=1e-2, weight_decay=0.0)
    hist = [net.relational_link_train_step(dec, t, opt) for _ in range(150)]
    loss, correct, count, _, _ = net.relational_link_evaluate(dec, t)
    assert count == 3000 and correct / count >= 0.9, (hist[0], hist[-1], correct / count)
    # the dot-product decoder on the same pairs: one score per pair, labelled 1 once and 0 once
    net2 = D.RGCN(alg, [(f, 16), (16, 16)], num_relations=R, aggr="mean")
    for l, Pp in enumerate(ro.random_params([(f, 16), (16, 16)], R, np.random.default_rng(SEED + 42), scale=0.5)):
        for k, vv in Pp.items():
            net2.set_param(l, k, vv)
    net2.set_input(np.vstack([X, np.zeros((net2.buffer_shape(0)[0] - N, f))]))
    lt = D.LinkTargets(net2, D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(
        N, N, np.concatenate([u, u]), np.concatenate([v, v]), np.concatenate([np.ones(1500), np.zeros(1500)])), f, 1))
    opt2 = D.AdamW(lr=1e-2, weight_decay=0.0)
    for _ in range(150):
        net2.link_train_step(lt, opt2)
    _, c2, n2, _ = net2.link_evaluate(lt)
    assert n2 == 3000 and c2 / n2 <= 0.5
