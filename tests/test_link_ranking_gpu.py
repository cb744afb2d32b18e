"""Filtered link ranking on the GPU (include/hnh/link_ranking.hpp, csrc/link_ranking.cu): the count, query and pair
kernels against numpy -- exactly on integer-valued operands, and on float operands through the pair path, which must
cancel the count path exactly -- at the table and odd widths, off the 64-tile, past one resident wave, with odd leading
dimensions and misaligned operands, and with exact ties; then net.link_rank on R-GCN (plain and with bases) with a
trained DistMult decoder and on GraphSAGE without one, against tests/link_ranking_oracle.py exactly; duplicate
queries, hub filters, every refusal, and a learning check.  Then integer-valued models r = 40001 to 262145 wide
(tests/link_ranking_cases.py), ranked in one to three query chunks and on all five layouts, exactly against
tests/link_ranking_oracle.matmul_ranks; every model on the float path, by dot product and two with DistMult; and
link_rank after a train step (stale activations) and after a dropout step."""
import math

import numpy as np
import pytest
import torch

from distributed_sddmm_b200 import driver as D
from distributed_sddmm_b200 import lib
from tests import gin_oracle as go
from tests import graph_sage_oracle as so
from tests import link_ranking_cases as lrc
from tests import link_ranking_oracle as lro
from tests import rgcn_basis_oracle as bo
from tests import rgcn_oracle as ro
from tests.test_link_prediction_gpu import _dev_rows

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
SEED = 0xC0FFEE + 433


@pytest.fixture(scope="module")
def world():
    D.world_init("self")
    yield
    D.world_finalize()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _ok(rc):
    assert rc == 0, lib().hnh_last_error_string()


# ---- the kernels ----------------------------------------------------------------------------------------------------------
def _ops(Z, Q, ld, offset):
    ldz, ldq = ld or (Z.shape[1], Q.shape[1])
    zb, qb = _dev_rows(Z, ldz, offset), _dev_rows(Q, ldq, offset)
    return (zb.data_ptr() + 8 * offset, ldz), (qb.data_ptr() + 8 * offset, ldq), (zb, qb)


def run_count(Z, Q, s_true, ld=None, offset=0, counts=None):
    """hnh_rank_count_f64: (gt, ge) as numpy int64, added to `counts` (2 x n_q, default zeros)."""
    (zp, ldz), (qp, ldq), keep = _ops(Z, Q, ld, offset)
    st = torch.from_numpy(np.asarray(s_true, np.float64)).to(DEV)
    c = torch.from_numpy(np.zeros((2, len(Q)), np.int64) if counts is None else counts.copy()).to(DEV)
    _ok(lib().hnh_rank_count_f64(zp, ldz, len(Z), qp, ldq, len(Q), Z.shape[1], st.data_ptr(), c[0].data_ptr(), c[1].data_ptr(),
                                 _st()))
    torch.cuda.synchronize()
    return c.cpu().numpy()


def run_pairs(Z, Q, pq, prow, s_true=None, counts=None, ld=None, offset=0):
    """hnh_rank_pairs_f64: (scores, counts after the subtraction, or None)."""
    (zp, ldz), (qp, ldq), keep = _ops(Z, Q, ld, offset)
    a, b = (torch.from_numpy(np.asarray(x, np.int64)).to(DEV) for x in (pq, prow))
    sc = torch.full((len(pq) + 1,), math.nan, dtype=torch.float64, device=DEV)
    st = c = None
    if counts is not None:
        st = torch.from_numpy(np.asarray(s_true, np.float64)).to(DEV)
        c = torch.from_numpy(counts.copy()).to(DEV)
    p = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    _ok(lib().hnh_rank_pairs_f64(zp, ldz, len(Z), qp, ldq, len(Q), Z.shape[1], a.data_ptr(), b.data_ptr(), len(pq), sc.data_ptr(),
                                 p(st), p(c[0]) if c is not None else None, p(c[1]) if c is not None else None, _st()))
    torch.cuda.synchronize()
    assert torch.isnan(sc[-1])
    return sc[:-1].cpu().numpy(), c.cpu().numpy() if c is not None else None


def np_counts(Z, Q, s_true):
    S = Z @ Q.T  # rows x n_q
    return np.stack([(S > s_true[None, :]).sum(0), (S >= s_true[None, :]).sum(0)]).astype(np.int64)


def integer_case(rng, rows, n_q, r):
    """Small-integer operands: every score is exact in fp64, and there are many ties.  s_true is a score of the
    query's own column (a tie with at least one row) or a value between scores."""
    Z = rng.integers(-3, 4, (rows, r)).astype(np.float64)
    Q = rng.integers(-3, 4, (n_q, r)).astype(np.float64)
    S = Z @ Q.T
    st = S[rng.integers(0, rows, n_q), np.arange(n_q)] + rng.choice([0.0, 0.5, -0.5], n_q)
    return Z, Q, st


def check_integer(Z, Q, st, **kw):
    got = run_count(Z, Q, st, **kw)
    assert np.array_equal(got, np_counts(Z, Q, st))
    assert np.array_equal(run_count(Z, Q, st, **kw), got)  # bit-identical repeats
    return got


def check_cancel(rng, Z, Q, **kw):
    """Float operands: s_true from the pair path at a random row; the count minus every (q, row) pair is exactly 0."""
    rows, n_q = len(Z), len(Q)
    own = rng.integers(0, rows, n_q)
    st, _ = run_pairs(Z, Q, np.arange(n_q), own, **kw)
    S = Z @ Q.T
    bound = np.abs(Z) @ np.abs(Q).T
    assert (np.abs(st - S[own, np.arange(n_q)]) <= 1e-13 * bound[own, np.arange(n_q)] + 1e-300).all()
    counts = run_count(Z, Q, st, **kw)
    # away from rounding, the counts are numpy's
    far = np.abs(S - st[None, :]) > 1e-12 * bound
    for k, above in enumerate((S > st[None, :], S >= st[None, :])):
        assert ((counts[k] >= (above & far).sum(0)) & (counts[k] <= (above | ~far).sum(0))).all()
    assert (counts[1] >= 1).all()  # the true row itself
    pq, prow = np.repeat(np.arange(n_q), rows), np.tile(np.arange(rows), n_q)
    sc, left = run_pairs(Z, Q, pq, prow, st, counts, **kw)
    assert not left.any(), left
    assert np.array_equal(sc.reshape(n_q, rows)[np.arange(n_q), own], st)  # the same pair, the same bits
    return counts


WIDTHS = list(range(1, 18)) + [63, 64, 65, 127, 128, 129, 500, 513]


@pytest.mark.parametrize("r", WIDTHS)
def test_rank_count_matches_numpy(world, r):
    rng = np.random.default_rng(SEED + r)
    check_integer(*integer_case(rng, 200, 130, r))
    check_cancel(rng, rng.standard_normal((150, r)), rng.standard_normal((70, r)))


@pytest.mark.parametrize("r", [1, 5, 64, 129, 513])
def test_rank_kernels_odd_ld_and_misaligned(world, r):
    rng = np.random.default_rng(SEED + 3 * r)
    for ld, offset in (((r + 1, r), 0), ((r, r + 3), 0), ((r, r), 1), ((r + 2, r + 1), 1)):
        check_integer(*integer_case(rng, 97, 65, r), ld=ld, offset=offset)
        check_cancel(rng, rng.standard_normal((97, r)), rng.standard_normal((65, r)), ld=ld, offset=offset)


@pytest.mark.parametrize("r,rows,n_q", [(4, 70001, 193), (64, 20000, 500), (513, 4100, 1100)])
def test_rank_kernels_past_one_wave(world, r, rows, n_q):
    """More 64 x 64 tiles than 132 SMs x 8 CTAs hold at once."""
    assert ((rows + 63) // 64) * ((n_q + 63) // 64) > 132 * 8
    rng = np.random.default_rng(SEED + rows)
    check_integer(*integer_case(rng, rows, n_q, r))
    if rows * n_q <= 5_000_000:
        check_cancel(rng, rng.standard_normal((rows, r)) / 4, rng.standard_normal((n_q, r)) / 4)


@pytest.mark.parametrize("r", [3, 64, 500])
def test_rank_ties_at_every_fragment_position(world, r):
    """Copies of row 5 at another row group (6), another DMMA tile of the warp (13), the other warp row half (37), and
    other CTA tiles (100, 190); copies of query 3 at another column pair (4), another DMMA tile (11), the other warp
    column half (40) and another CTA tile (70).  Every copy scores the same bits, so each ties exactly."""
    rng = np.random.default_rng(SEED + 7 * r)
    Z, Q = rng.standard_normal((200, r)), rng.standard_normal((90, r))
    dup_rows, dup_q = [6, 13, 37, 100, 190], [4, 11, 40, 70]
    Z[dup_rows], Q[dup_q] = Z[5], Q[3]
    st, _ = run_pairs(Z, Q, np.arange(90), np.full(90, 5))
    c = run_count(Z, Q, st)
    assert (c[1] - c[0] == 1 + len(dup_rows)).all()  # the true row and its copies tie, nothing else does
    assert all(np.array_equal(c[:, 3], c[:, q]) for q in dup_q)
    sc, _ = run_pairs(Z, Q, np.repeat(np.arange(90), 6), np.tile([5] + dup_rows, 90))
    assert (sc.reshape(90, 6) == st[:, None]).all()
    # all-zero embeddings: every score is 0 and ties with the true one
    z0 = np.zeros((131, r))
    c0 = run_count(z0, Q, np.zeros(90))
    assert not c0[0].any() and (c0[1] == 131).all()


def test_rank_queries_kernel(world):
    rng = np.random.default_rng(SEED + 9)
    rows, r, R, n_q, row0 = 50, 7, 4, 120, 100
    Z, Dt = rng.standard_normal((rows, r)), rng.standard_normal((R, r))
    anchors = rng.integers(80, 170, n_q)  # some before, some past this block
    rels = rng.integers(-1, R + 1, n_q)  # some outside [0, R)
    for with_d in (True, False):
        Q = torch.full((n_q * (r + 2) + 1,), math.nan, dtype=torch.float64, device=DEV)
        z, d = (torch.from_numpy(x).to(DEV) for x in (Z, Dt))
        a, b = (torch.from_numpy(x.astype(np.int64)).to(DEV) for x in (anchors, rels))
        _ok(lib().hnh_rank_queries_f64(Q.data_ptr(), r + 2, n_q, z.data_ptr(), r, row0, rows, a.data_ptr(), b.data_ptr(),
                                       d.data_ptr() if with_d else None, r, R, r, _st()))
        torch.cuda.synchronize()
        got = Q[:-1].view(n_q, r + 2).cpu().numpy()
        own = (anchors >= row0) & (anchors < row0 + rows)
        want = np.zeros((n_q, r))
        want[own] = Z[anchors[own] - row0]
        if with_d:
            ok = own & (rels >= 0) & (rels < R)
            want[ok] *= Dt[rels[ok]]
            want[own & ~ok] = 0.0
        assert np.array_equal(got[:, :r], want) and np.isnan(got[:, r:]).all()


def test_rank_kernel_argument_checks(world):
    L = lib()
    assert L.hnh_rank_count_f64(None, 4, 10, None, 4, 10, 0, None, None, None, None) != 0  # r = 0
    assert L.hnh_rank_count_f64(None, 3, 10, None, 4, 10, 4, None, None, None, None) != 0  # ldz < r
    assert L.hnh_rank_count_f64(None, 4, 0, None, 4, 10, 4, None, None, None, None) == 0  # nothing to count
    assert L.hnh_rank_pairs_f64(None, 4, 10, None, 4, 10, 4, None, None, -1, None, None, None, None, None) != 0


# ---- the model level ------------------------------------------------------------------------------------------------------
def _kg(rng, N, R, n):
    h, rr, t = rng.integers(0, N, n), rng.integers(0, R, n), rng.integers(0, N, n)
    return h.astype(np.int64), rr.astype(np.int64), t.astype(np.int64)


def rgcn_kg(B, seed, N=160, R=3, f=6, r=8):
    rng = np.random.default_rng(seed)
    train, valid, test = _kg(rng, N, R, 900), _kg(rng, N, R, 60), _kg(rng, N, R, 60)
    alg = D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, train[0], train[2], train[1].astype(np.float64)), f, 1)
    net = D.RGCN(alg, [(f, 16), (16, r)], num_relations=R, num_bases=B)
    params = bo.random_params([(f, 16), (16, r)], R, B, rng) if B else ro.random_params([(f, 16), (16, r)], R, rng)
    for l, P in enumerate(params):
        for k, v in P.items():
            net.set_param(l, k, v)
    net.set_input(np.vstack([rng.uniform(-1, 1, (N, f)), np.zeros((net.buffer_shape(0)[0] - N, f))]))
    dec = D.DistMultDecoder(net, R)
    dec.set_param("rel", rng.uniform(-1, 1, (R, r)))
    # a few relational train steps, negatives by corrupting tails
    neg = (train[0], train[1], rng.integers(0, N, len(train[0])))
    mk = lambda t: D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, t[0], t[2], t[1].astype(np.float64)), f, 1)  # noqa: E731
    a_pos, a_neg = mk(train), mk(neg)
    targets = D.RelationalLinkTargets(net, a_pos, a_neg, R)
    opt = D.AdamW(lr=1e-2)
    for _ in range(5):
        net.relational_link_train_step(dec, targets, opt)
    return dict(N=N, R=R, net=net, dec=dec, alg=alg, train=train, valid=valid, test=test, keep=(a_pos, a_neg, targets))


@pytest.mark.parametrize("B", [None, 2])
def test_rgcn_distmult_ranks_match_the_oracle(world, B):
    K = rgcn_kg(B, SEED + 20 + (B or 0))
    net, dec, N, R = K["net"], K["dec"], K["N"], K["R"]
    rng = np.random.default_rng(SEED + 21)
    # a hub (head, relation) whose filter holds more than half the nodes, and one whose filter holds every node
    hub = (np.full(100, 7), np.full(100, 1), rng.permutation(N)[:100])
    full = (np.full(N, 9), np.full(N, 2), np.arange(N))
    known = [K["train"], K["valid"], K["test"], hub, full]
    ranking = D.LinkRanking(net, tuple(np.concatenate(x) for x in zip(*known)), R)
    q = tuple(np.concatenate([a, a[:5], b[:3], c[:2]]) for a, b, c in zip(K["test"], hub, full))  # duplicates, hubs
    res = net.link_rank(ranking, q, decoder=dec)
    z, rel = net.buffer(len(net.layers))[:N], dec.param("rel")
    mrr, t, h, st, sh = lro.filtered_ranks(z, rel, q, known, N)
    assert lro.separated(st, sh, q)
    assert np.array_equal(res.tail_ranks, t) and np.array_equal(res.head_ranks, h)
    assert res.mrr == pytest.approx(mrr, rel=1e-14)
    n = len(K["test"][0])
    assert np.array_equal(res.tail_ranks[n:n + 5], res.tail_ranks[:5]) and np.array_equal(res.head_ranks[n:n + 5], res.head_ranks[:5])
    assert (res.tail_ranks[-2:] == 1.0).all()  # every node is a known tail of (9, 2)
    # every query is in F: PyG's loop gives the same ranks (a sample of queries, the loop is slow)
    sample = tuple(a[::7] for a in q)
    _, lt, lh = lro.compute_mrr_loop(z, lro.decoder_of(rel), sample, known, N)
    assert np.array_equal(lt, res.tail_ranks[::7]) and np.array_equal(lh, res.head_ranks[::7])
    assert res.hits_at(10) == pytest.approx(((t <= 10).sum() + (h <= 10).sum()) / (2 * len(t)))
    again = net.link_rank(ranking, q, decoder=dec)
    assert np.array_equal(again.tail_ranks, res.tail_ranks) and again.mrr == res.mrr
    # an empty filter: the raw ranks, the true entity counted once
    raw = net.link_rank(D.LinkRanking(net, ([], [], []), R), q, decoder=dec)
    _, rt, rh, _, _ = lro.filtered_ranks(z, rel, q, [], N)
    assert np.array_equal(raw.tail_ranks, rt) and np.array_equal(raw.head_ranks, rh)


def sage_net(seed, N=150, f=5, r=6, dup=(20, 21, 22, 140)):
    """GraphSAGE whose nodes `dup` have no entries and one input row: their output rows are the same bits."""
    rng = np.random.default_rng(seed)
    rows, cols = rng.integers(0, N, 700), rng.integers(0, N, 700)
    keep = ~np.isin(rows, dup)
    rows, cols = rows[keep], cols[keep]
    alg = D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, rows, cols, np.ones(len(rows))), f, 1)
    net = D.GraphSAGE(alg, [(f, 12), (12, r)], aggr="mean")
    for l, P in enumerate(so.random_params([(f, 12), (12, r)], rng)):
        for k, v in P.items():
            net.set_param(l, k, v)
    X = rng.uniform(-1, 1, (N, f))
    X[list(dup)] = X[dup[0]]
    net.set_input(np.vstack([X, np.zeros((net.buffer_shape(0)[0] - N, f))]))
    return net, alg, N


def test_graph_sage_dot_product_ranks_match_the_oracle(world):
    net, alg, N = sage_net(SEED + 30)
    rng = np.random.default_rng(SEED + 31)
    known = [(rng.integers(0, N, 500), np.zeros(500, np.int64), rng.integers(0, N, 500))]
    q = (np.concatenate([known[0][0][:80], [20, 3, 21]]), np.zeros(83, np.int64), np.concatenate([known[0][2][:80], [5, 22, 140]]))
    known.append(tuple(a[80:] for a in q))  # the extra queries are known too
    ranking = D.LinkRanking(net, tuple(np.concatenate(x) for x in zip(*known)))
    res = net.link_rank(ranking, q)
    z = net.buffer(len(net.layers))[:N]
    assert np.array_equal(z[20], z[21]) and np.array_equal(z[20], z[140])
    mrr, t, h, st, sh = lro.filtered_ranks(z, np.ones((1, z.shape[1])), q, known, N)
    assert lro.separated(st, sh, q)
    assert np.array_equal(res.tail_ranks, t) and np.array_equal(res.head_ranks, h)
    assert (t != np.round(t)).any() or (h != np.round(h)).any()  # the copies tie: half ranks


def test_link_rank_refusals(world):
    K = rgcn_kg(None, SEED + 40, N=100)
    net, dec, N, R = K["net"], K["dec"], K["N"], K["R"]
    pad = net.buffer_shape(len(net.layers))[0]
    F = K["train"]
    for bad, what in ((([N], [0], [1]), "outside"), (([0], [0], [-1]), "outside"), (([0], [R], [1]), "relation"),
                      (([0], [-1], [1]), "relation")):
        with pytest.raises(RuntimeError, match=what):
            D.LinkRanking(net, bad, R)
    if pad > N:
        with pytest.raises(RuntimeError, match="outside"):
            D.LinkRanking(net, ([0], [0], [pad - 1]), R)
    with pytest.raises(RuntimeError, match="relation count"):
        D.LinkRanking(net, F, 0)
    ranking = D.LinkRanking(net, F, R)
    q = K["test"]
    for bad in (([N], [0], [1]), ([0], [R], [1]), ([0], [0], [-3])):
        with pytest.raises(RuntimeError, match="query"):
            net.link_rank(ranking, bad, decoder=dec)
    with pytest.raises(RuntimeError, match="1 relation"):
        net.link_rank(ranking, q)  # no decoder with R = 3
    with pytest.raises(RuntimeError, match="relations"):
        net.link_rank(D.LinkRanking(net, F, R + 1), q, decoder=dec)
    other = rgcn_kg(None, SEED + 41, N=100)
    with pytest.raises(RuntimeError, match="ranking was made for another"):
        net.link_rank(D.LinkRanking(other["net"], F, R), q, decoder=dec)
    with pytest.raises(RuntimeError, match="decoder was made for another"):
        net.link_rank(ranking, q, decoder=other["dec"])
    narrow = D.RGCN(net.alg, [(6, 5)], num_relations=R)  # the same algorithm object, an output 5 wide
    with pytest.raises(RuntimeError, match="wide"):
        net.link_rank(ranking, q, decoder=D.DistMultDecoder(narrow, R))
    with pytest.raises(ValueError, match="entries"):
        net.link_rank(ranking, ([0, 1], [0], [1]), decoder=dec)
    with pytest.raises(TypeError):
        net.link_rank(F, q, decoder=dec)
    res = net.link_rank(ranking, ([], [], []), decoder=dec)
    assert res.mrr == 0.0 and len(res.tail_ranks) == 0


# ---- learning ----------------------------------------------------------------------------------------------------------
def test_filtered_mrr_rises_with_training(world):
    """The learning-check data of tests/test_distmult_gpu.py: relation 0 joins nodes of one community, relation 1
    nodes of different ones.  R-GCN with DistMult trained on 1500 triples ranks 300 held-out triples.  One recorded run
    on an H100 gave a filtered MRR of 0.052 before training and 0.082 after, Hits@10 0.10 and 0.17; the margins below
    sit under those ratios."""
    N, R, f = 128, 2, 8
    rng = np.random.default_rng(SEED + 50)
    comm = np.arange(N) % 2
    from oracle import hnh_oracle as orc
    rows, cols, _ = orc.er_tuples(7, 6, SEED + 51)
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    alg = D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, rows, cols, (comm[rows] != comm[cols]).astype(np.float64)), f, 1)
    net = D.RGCN(alg, [(f, 16), (16, 16)], num_relations=R, aggr="mean")
    for l, Pp in enumerate(ro.random_params([(f, 16), (16, 16)], R, rng, scale=0.5)):
        for k, v in Pp.items():
            net.set_param(l, k, v)
    net.set_input(np.vstack([rng.standard_normal((N, f)), np.zeros((net.buffer_shape(0)[0] - N, f))]))
    u, v = rng.integers(0, N, 1800), rng.integers(0, N, 1800)
    rel = (comm[u] != comm[v]).astype(np.int64)
    train, held = (u[:1500], rel[:1500], v[:1500]), (u[1500:], rel[1500:], v[1500:])
    mk = lambda rr: D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, train[0], train[2], rr), f, 1)  # noqa: E731
    a_pos, a_neg = mk(train[1].astype(np.float64)), mk(1.0 - train[1])
    dec = D.DistMultDecoder(net, R)
    dec.set_param("rel", rng.uniform(-0.5, 0.5, (R, 16)))
    ranking = D.LinkRanking(net, (u, rel, v), R)
    before = net.link_rank(ranking, held, decoder=dec)
    t = D.RelationalLinkTargets(net, a_pos, a_neg, R)
    opt = D.AdamW(lr=1e-2, weight_decay=0.0)
    for _ in range(150):
        net.relational_link_train_step(dec, t, opt)
    after = net.link_rank(ranking, held, decoder=dec)
    print(f"filtered MRR before {before.mrr:.4f} after {after.mrr:.4f}, Hits@10 {before.hits_at(10):.3f} -> {after.hits_at(10):.3f}")
    assert after.mrr >= 1.3 * before.mrr and after.hits_at(10) >= before.hits_at(10) + 0.04, (before, after)


# ---- wide integer-valued models: several query chunks, exactly --------------------------------------------------------
def integer_net(model, r, M, seed, alg_name="15d_fusion1", R=None, nonneg=False):
    """An integer-valued model of tests/link_ranking_cases.py (GraphSAGE sum, GIN eps = 0, R-GCN sum with and without
    bases) r wide on M nodes, its input set, and a DistMult decoder of R relations (None: no decoder)."""
    rows, cols, rels = lrc.graph(M, seed)
    vals = rels if model.startswith("rgcn") else np.ones(len(rows))
    alg = D.Algorithm(alg_name, D.SpmatLocal.from_tuples(M, M, rows, cols, vals), lrc.F_IN, 1)
    L = lrc.layers(model, r)
    net = {"sage": lambda: D.GraphSAGE(alg, L, aggr="sum"), "gin": lambda: D.GIN(alg, L, eps=0.0),
           "rgcn": lambda: D.RGCN(alg, L, lrc.RELS, aggr="sum"),
           "rgcn_bases": lambda: D.RGCN(alg, L, lrc.RELS, aggr="sum", num_bases=lrc.BASES)}[model]()
    rng = np.random.default_rng(seed + 1)
    for l in range(len(L)):
        for name in net.param_names():
            if name != "eps":
                net.set_param(l, name, lrc.integer_param(net.param_shape(l, name), rng, nonneg))
    X = lrc.integer_input(M, seed + 2, nonneg)
    net.set_input(np.vstack([X, np.zeros((net.buffer_shape(0)[0] - M, X.shape[1]))]))
    dec = rel = None
    if R:
        dec = D.DistMultDecoder(net, R)
        rel = lrc.relation_table(R, r, seed + 3, nonneg)
        dec.set_param("rel", rel)
    return net, alg, dec, (rel if R else np.ones((1, r)))


def candidates(F, R, M, q, tail):
    """|C| per query: the nodes other than the true entity and outside the filter."""
    keys = lro.filter_keys([F], R, M)
    v = np.arange(M)
    h, rr, t = q
    k = ((h * R + rr)[:, None] * M + v[None, :]) if tail else ((v[None, :] * R + rr[:, None]) * M + t[:, None])
    c = ~np.isin(k, keys)
    c[np.arange(len(h)), t if tail else h] = False
    return c.sum(1)


def check_exact(res, z, rel, q, known, M):
    """link_rank's result against the exact oracle on the integer-valued output z."""
    assert np.array_equal(z, np.round(z)), "the output is not integer-valued"
    assert lro.integer_bound(z, rel) < 2.0 ** 43  # a 2^10 margin below 2^53
    mrr, t, h, st, sh = lro.matmul_ranks(z, rel, q, known, M)
    assert np.array_equal(res.tail_ranks, t) and np.array_equal(res.head_ranks, h)
    assert res.mrr == pytest.approx(mrr, rel=1e-14)
    for k in (1, 3, 10):
        assert res.hits_at(k) == ((t <= k).sum() + (h <= k).sum()) / (2 * len(t))
    return t, h, st, sh


@pytest.mark.parametrize("name", sorted(lrc.WIDE))
def test_wide_integer_ranks_are_exact_across_chunks(world, name):
    cfg = lrc.WIDE[name]
    M, r, R, n_q = cfg["M"], cfg["r"], cfg["R"], cfg["n_q"]
    seed = lrc.case_seed(name)
    net, alg, dec, rel = integer_net(cfg["model"], r, M, seed, R=R)
    chunk = lrc.chunk_of(r, n_q)
    F, q, lonely, hub, edges = lrc.queries(M, R or 1, n_q, chunk, seed + 4)
    ranking = D.LinkRanking(net, F, R or 1)
    res = net.link_rank(ranking, q, decoder=dec)
    z = net.buffer(len(net.layers))[:M]
    iso = lrc.isolated(M)
    assert all(np.array_equal(z[iso[0]], z[i]) for i in iso[1:])  # copies: their scores tie exactly
    t, h, st, sh = check_exact(res, z, rel, q, [F], M)
    assert (st[:, iso] == st[:, iso[:1]]).all()
    again = net.link_rank(ranking, q, decoder=dec)
    assert np.array_equal(again.tail_ranks, res.tail_ranks) and np.array_equal(again.head_ranks, res.head_ranks)
    assert again.mrr == res.mrr
    for e in edges:  # one query on both sides of a chunk edge
        assert (q[0][e - 1], q[1][e - 1], q[2][e - 1]) == (q[0][e], q[1][e], q[2][e])
        assert t[e - 1] == t[e] and h[e - 1] == h[e]
    assert (t[(q[0] == hub) & (q[1] == 0)] == 1.0).all()  # every node is a known tail of (hub, 0)
    if R:
        zero = q[1] == lrc.ZERO_REL  # every score is 0: every candidate ties with the true entity
        assert zero.any() and not (q[1] == lrc.UNUSED_REL).any()
        assert np.array_equal(t[zero], (1 + (candidates(F, R, M, q, True)[zero] + 1)) / 2)
        assert np.array_equal(h[zero], (1 + (candidates(F, R, M, q, False)[zero] + 1)) / 2)
    assert ((st == st[np.arange(n_q), q[2]][:, None]).sum(1) > 1).any()  # candidates tie with the true tail
    # an empty filter: the raw ranks
    raw = net.link_rank(D.LinkRanking(net, ([], [], []), R or 1), q, decoder=dec)
    check_exact(raw, z, rel, q, [], M)


ALL_LAYOUTS = ["15d_fusion1", "15d_fusion2", "15d_sparse", "25d_dense_replicate", "25d_sparse_replicate"]


def test_integer_ranks_on_every_layout_at_p1(world):
    """The five layouts hold full rows at p = 1: the same output, the same ranks."""
    cfg = lrc.WIDE["rgcn_r40001_distmult"]
    M, r, R, n_q = cfg["M"], cfg["r"], cfg["R"], cfg["n_q"]
    seed = SEED + 70
    F, q, _, _, _ = lrc.queries(M, R, n_q, lrc.chunk_of(r, n_q), seed + 4)
    z0 = want = None
    for name in ALL_LAYOUTS:
        net, alg, dec, rel = integer_net(cfg["model"], r, M, seed, alg_name=name, R=R)
        res = net.link_rank(D.LinkRanking(net, F, R), q, decoder=dec)
        z = net.buffer(len(net.layers))[:M]
        if z0 is None:
            z0, want = z, check_exact(res, z, rel, q, [F], M)
        assert np.array_equal(z, z0), name
        assert np.array_equal(res.tail_ranks, want[0]) and np.array_equal(res.head_ranks, want[1]), name


# ---- every model, on the float path ----------------------------------------------------------------------------------
FLOAT_MODELS = ["gat_leaky", "gat_softmax", "gat_additive", "gat_gatv2", "gt_plain", "gt_edge_beta_ffn", "sage_mean",
                "sage_sum", "sage_max", "pna", "gin", "gine"]
N_FLOAT, F_FLOAT = 150, 6


def float_net(kind, seed):
    """A model of kind with every parameter random, its input (and edge attributes) set; output 6 wide."""
    rng = np.random.default_rng(seed)
    N, f = N_FLOAT, F_FLOAT
    rows, cols = rng.integers(0, N, 800), rng.integers(0, N, 800)
    alg = D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, rows, cols, np.ones(len(rows))), f, 1)
    if kind.startswith("gat"):
        L = [(f, 4, 2), (8, 6, 1)]
        net = D.GAT(alg, L, attention=kind[4:])
        for l, (fi, d, H) in enumerate(L):
            for hd in range(H):
                net.set_weight(l, hd, rng.uniform(-1, 1, (fi, d)) / np.sqrt(fi))
                net.set_attention_vectors(l, hd, rng.uniform(-1, 1, d), rng.uniform(-1, 1, d))
    else:
        if kind.startswith("gt"):
            full = kind == "gt_edge_beta_ffn"
            L = [(f, 4, 2), (8, 3, 2)]
            net = D.GraphTransformer(alg, L, edge_dim=3 if full else 0, beta=full, ffn_ratio=2 if full else 0)
        elif kind.startswith("sage"):
            L = [(f, 10), (10, 6)]
            net = D.GraphSAGE(alg, L, aggr=kind[5:])
        elif kind == "pna":
            L = [(f, 10), (10, 6)]
            net = D.PNA(alg, L, deg=np.bincount(np.bincount(rows, minlength=N)))
        else:
            L = [(f, 10, 8), (8, 10, 6)]
            net = D.GIN(alg, L, edge_dim=3 if kind == "gine" else 0, eps=0.25)
        for l in range(len(L)):
            for name in net.param_names():
                shape = net.param_shape(l, name)
                net.set_param(l, name, rng.uniform(-1, 1, shape) / (np.sqrt(shape[0]) if len(shape) == 2 else 2.0))
        if getattr(net, "edge_dim", 0):
            net.set_edge_attributes(go.attr_of(*alg.entry_coordinates("A"), 3), go.attr_of(*alg.entry_coordinates("B"), 3))
    X = rng.uniform(-1, 1, (N, f))
    net.set_input(np.vstack([X, np.zeros((net.buffer_shape(0)[0] - N, f))]))
    return net, alg, rows, cols


def float_queries(rng, N, R, n=120):
    known = [_kg(rng, N, R, 600)]
    q = _kg(rng, N, R, n)
    known.append(tuple(a[: n // 2] for a in q))
    return known, q


def check_float(res, z, rel, q, known, N):
    mrr, t, h, st, sh = lro.matmul_ranks(z, rel, q, known, N)
    assert lro.separated(st, sh, q)
    assert np.array_equal(res.tail_ranks, t) and np.array_equal(res.head_ranks, h)
    assert res.mrr == pytest.approx(mrr, rel=1e-14)


@pytest.mark.parametrize("kind", FLOAT_MODELS)
def test_every_model_dot_product_ranks_match_the_oracle(world, kind):
    net, alg, _, _ = float_net(kind, SEED + 80 + len(kind))
    rng = np.random.default_rng(SEED + 81)
    known, q = float_queries(rng, N_FLOAT, 1)
    ranking = D.LinkRanking(net, tuple(np.concatenate(x) for x in zip(*known)))
    res = net.link_rank(ranking, q)
    z = net.buffer(len(net.layers))[:N_FLOAT]
    assert np.abs(z).max() > 0
    check_float(res, z, np.ones((1, z.shape[1])), q, known, N_FLOAT)


@pytest.mark.parametrize("kind", ["gt_plain", "gine"])
def test_distmult_ranks_of_other_models_match_the_oracle(world, kind):
    net, alg, _, _ = float_net(kind, SEED + 90 + len(kind))
    rng = np.random.default_rng(SEED + 91)
    R = 2
    dec = D.DistMultDecoder(net, R)
    dec.set_param("rel", rng.uniform(-1, 1, (R, 6)))
    known, q = float_queries(rng, N_FLOAT, R)
    res = net.link_rank(D.LinkRanking(net, tuple(np.concatenate(x) for x in zip(*known)), R), q, decoder=dec)
    check_float(res, net.buffer(len(net.layers))[:N_FLOAT], dec.param("rel"), q, known, N_FLOAT)


def _link_targets(net, rng, N):
    tr, tc = rng.integers(0, N, 400), rng.integers(0, N, 400)
    algT = D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, tr, tc, rng.choice([0.0, 1.0], 400)), F_FLOAT, 1)
    return algT, D.LinkTargets(net, algT)


@pytest.mark.parametrize("kind", ["sage_mean", "gin", "gat_softmax"])
def test_link_rank_after_a_train_step_ranks_the_updated_model(world, kind):
    """A train step leaves the activations of the parameters before its update: link_rank must run the forward."""
    net, alg, _, _ = float_net(kind, SEED + 100 + len(kind))
    rng = np.random.default_rng(SEED + 101)
    known, q = float_queries(rng, N_FLOAT, 1)
    ranking = D.LinkRanking(net, tuple(np.concatenate(x) for x in zip(*known)))
    net.forward()
    before = net.buffer(len(net.layers))
    algT, t = _link_targets(net, rng, N_FLOAT)
    net.link_train_step(t, D.AdamW(lr=5e-2))
    assert np.array_equal(net.buffer(len(net.layers)), before)  # the buffer still holds the old activations
    res = net.link_rank(ranking, q)
    z = net.buffer(len(net.layers))
    assert not np.array_equal(z, before)
    net.forward()
    assert np.array_equal(net.buffer(len(net.layers)), z)  # bit for bit an explicit forward's
    check_float(res, z[:N_FLOAT], np.ones((1, z.shape[1])), q, known, N_FLOAT)


def test_link_rank_after_a_dropout_step_ranks_without_dropout(world):
    net, alg, _, _ = float_net("gt_plain", SEED + 110)
    rng = np.random.default_rng(SEED + 111)
    known, q = float_queries(rng, N_FLOAT, 1)
    ranking = D.LinkRanking(net, tuple(np.concatenate(x) for x in zip(*known)))
    algT, t = _link_targets(net, rng, N_FLOAT)
    net.link_train_step(t, D.AdamW(lr=1e-2), dropout=0.4, seed=9)
    res = net.link_rank(ranking, q)
    z = net.buffer(len(net.layers))
    net.forward(dropout=0.4, seed=9)
    assert not np.array_equal(net.buffer(len(net.layers)), z)  # dropout changes the output
    net.forward()
    assert np.array_equal(net.buffer(len(net.layers)), z)
    check_float(res, z[:N_FLOAT], np.ones((1, z.shape[1])), q, known, N_FLOAT)
