"""Filtered link ranking without a GPU: PyG's compute_mrr loop (tests/link_ranking_oracle.py) against the vectorised
definition the library implements, on small knowledge graphs with F = train + valid + test, the documented empty-F
difference, and the Hits@K helper of the Python results; the exact matmul oracle against both; and the claims of the
wide integer fixtures of tests/link_ranking_cases.py: chunk counts from the header's kRankChunkDoubles, the padded and
empty row blocks, the placements of ties and duplicates, and an integer bound far below 2^53."""
import numpy as np
import pytest

from tests import link_ranking_cases as lrc
from tests import link_ranking_oracle as lro

SEED = 0xC0FFEE + 431


def kg(rng, N, R, n):
    h, r, t = rng.integers(0, N, n), rng.integers(0, R, n), rng.integers(0, N, n)
    h[:12] = 3  # a hub (head, relation): many known tails
    r[:12] = R - 1
    return h, r, t


def splits(rng, N, R):
    train, valid, test = kg(rng, N, R, 300), kg(rng, N, R, 40), kg(rng, N, R, 40)
    return train, valid, test


@pytest.mark.parametrize("integer", [False, True])
@pytest.mark.parametrize("R", [1, 4])
def test_loop_and_vectorised_ranks_agree(R, integer):
    """Integer-valued embeddings make every score exact and give many ties; float ones give generic scores."""
    rng = np.random.default_rng(SEED + R + 10 * integer)
    N, r = 60, 5
    train, valid, test = splits(rng, N, R)
    z = rng.integers(-2, 3, (N, r)).astype(np.float64) if integer else rng.standard_normal((N, r))
    rel = rng.integers(-1, 2, (R, r)).astype(np.float64) if integer else rng.standard_normal((R, r))
    known = [train, valid, test]
    mrr, t, h = lro.compute_mrr_loop(z, lro.decoder_of(rel), test, known, N)
    vm, vt, vh, _, _ = lro.filtered_ranks(z, rel, test, known, N, chunk=7)
    assert np.array_equal(t, vt) and np.array_equal(h, vh)
    assert mrr == pytest.approx(vm, rel=1e-15)
    if integer:
        assert (t != np.round(t)).any()  # ties that split a rank into halves


def test_empty_filter_counts_the_true_entity_once():
    rng = np.random.default_rng(SEED + 1)
    N, R, r = 50, 3, 4
    _, _, test = splits(rng, N, R)
    z, rel = rng.standard_normal((N, r)), rng.standard_normal((R, r))
    _, t, h = lro.compute_mrr_loop(z, lro.decoder_of(rel), test, [], N)
    _, vt, vh, _, _ = lro.filtered_ranks(z, rel, test, [], N)
    # the loop keeps the true entity among its candidates and counts it a second time in the pessimistic rank
    assert np.array_equal(t, vt + 0.5) and np.array_equal(h, vh + 0.5)
    # raw ranks: 1 + the candidates above, with all N - 1 others as candidates
    s = ((z[test[0]] * rel[test[1]])[:, None, :] * z[None]).sum(-1)
    true = s[np.arange(len(test[0])), test[2]]
    assert np.array_equal(vt, ((s > true[:, None]).sum(1) + 1) + 0.0)


def test_every_candidate_filtered_gives_rank_one():
    rng = np.random.default_rng(SEED + 2)
    N, r = 30, 3
    z, rel = rng.standard_normal((N, r)), np.ones((1, r))
    full = (np.full(N, 4), np.zeros(N, np.int64), np.arange(N))  # (4, 0, v) is known for every v
    q = (np.array([4, 4]), np.array([0, 0]), np.array([7, 19]))
    _, t, _, _, _ = lro.filtered_ranks(z, rel, q, [full], N)
    _, lt, _ = lro.compute_mrr_loop(z, lro.decoder_of(rel), q, [full], N)
    assert np.array_equal(t, [1.0, 1.0]) and np.array_equal(lt, t)


def test_hits_at():
    from distributed_sddmm_b200.driver import LinkRanks
    res = LinkRanks(0.0, np.array([1.0, 1.5, 3.0, 10.0]), np.array([2.0, 2.5, 1.0, 11.0]))
    assert res.hits_at(1) == 2 / 8 and res.hits_at(2) == 4 / 8 and res.hits_at(3) == 6 / 8 and res.hits_at(10) == 7 / 8
    assert LinkRanks(0.0, np.zeros(0), np.zeros(0)).hits_at(3) == 0.0


# ---- the exact oracle ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("integer", [False, True])
@pytest.mark.parametrize("R", [1, 4])
def test_matmul_oracle_agrees_with_both_definitions(R, integer):
    rng = np.random.default_rng(SEED + 20 + R + 10 * integer)
    N, r = 60, 5
    train, valid, test = splits(rng, N, R)
    z = rng.integers(-2, 3, (N, r)).astype(np.float64) if integer else rng.standard_normal((N, r))
    rel = rng.integers(-1, 2, (R, r)).astype(np.float64) if integer else rng.standard_normal((R, r))
    known = [train, valid, test]
    mrr, t, h, st, sh = lro.filtered_ranks(z, rel, test, known, N, chunk=7)
    for chunk in (None, 1, 7, 1000):
        m2, t2, h2, st2, sh2 = lro.matmul_ranks(z, rel, test, known, N, chunk=chunk)
        assert np.array_equal(t, t2) and np.array_equal(h, h2)
        assert m2 == pytest.approx(mrr, rel=1e-15)
        if integer:
            assert np.array_equal(st, st2) and np.array_equal(sh, sh2)
        else:
            assert np.abs(st - st2).max() <= 1e-12 and np.abs(sh - sh2).max() <= 1e-12
    _, lt, lh = lro.compute_mrr_loop(z, lro.decoder_of(rel), test, known, N)
    assert np.array_equal(lt, t) and np.array_equal(lh, h)
    # an empty filter
    _, et, eh, _, _ = lro.filtered_ranks(z, rel, test, [], N)
    _, mt, mh, _, _ = lro.matmul_ranks(z, rel, test, [], N)
    assert np.array_equal(et, mt) and np.array_equal(eh, mh)


def test_matmul_oracle_is_exact_on_wide_integer_operands():
    """At r = 4097 with entries up to 50 the products reach 2^21 per term: integer sums, any order, the same bits."""
    rng = np.random.default_rng(SEED + 30)
    N, r, R = 40, 4097, 2
    z = rng.integers(-50, 51, (N, r)).astype(np.float64)
    z[[5, 17, 33]] = z[2]
    rel = rng.integers(-2, 3, (R, r)).astype(np.float64)
    q = (rng.integers(0, N, 30), rng.integers(0, R, 30), np.concatenate([[2, 5, 17], rng.integers(0, N, 27)]))
    _, t, h, st, _ = lro.matmul_ranks(z, rel, q, [], N, chunk=4)
    exact = [[sum(int(a) * int(b) * int(c) for a, b, c in zip(z[q[0][i]], rel[q[1][i]], z[v])) for v in range(N)] for i in range(3)]
    assert np.array_equal(st[:3], np.array(exact, np.float64))
    assert (st[:3][:, [2, 5, 17, 33]] == st[:3][:, [2]]).all()  # the copies tie
    assert lro.integer_bound(z, rel) < 2.0 ** 53


# ---- the fixtures of the wide GPU cases --------------------------------------------------------------------------------
def test_chunk_size_matches_the_header():
    assert lrc.rank_chunk_doubles() == 1 << 24
    assert lrc.chunk_of(16) == 1 << 20 and lrc.chunk_of(1 << 18) == 64 and lrc.chunk_of((1 << 18) + 1) == 64


@pytest.mark.parametrize("name", sorted(lrc.WIDE))
def test_wide_cases_reach_what_they_claim(name):
    cfg = lrc.WIDE[name]
    r, n_q, M = cfg["r"], cfg["n_q"], cfg["M"]
    chunk = lrc.chunk_of(r)
    want_chunk, n_chunks, partial = lrc.WIDE_REACHES[name]
    assert chunk == want_chunk and -(-n_q // chunk) == n_chunks and (n_q % chunk != 0) == partial
    if chunk == 64:
        assert lrc.rank_chunk_doubles() // r < 64  # the floor
    if r % 2:
        assert r % 64 != 0  # an odd width: the GEMMs pad K
    seed = lrc.case_seed(name)  # the instances the GPU test ranks
    F, q, lonely, hub, edges = lrc.queries(M, cfg["R"] or 1, n_q, chunk, seed + 4)
    assert edges == [k * chunk for k in range(1, n_chunks)]
    for e in edges:  # the same query on both sides of every chunk edge
        assert all(a[e - 1] == a[e] for a in q)
    iso = lrc.isolated(M)
    assert np.isin(q[2], iso).any() and (q[0] == q[2]).any()  # tie targets and self-loops
    assert ((q[0] == hub) & (q[1] == 0)).any() and set(F[2][(F[0] == hub) & (F[1] == 0)]) == set(range(M))
    assert (q[0] == lonely).any() and not ((F[0] == lonely) | (F[2] == lonely) & (F[0] != hub)).any()
    if cfg["R"]:
        assert (q[1] == lrc.ZERO_REL).any() and not (q[1] == lrc.UNUSED_REL).any()
        assert not lrc.relation_table(cfg["R"], 16, 0)[lrc.ZERO_REL].any()
    if M >= 201:
        assert len(set((iso // 64).tolist())) == len(iso)  # the copies sit in different 64-row tiles
    # the integer magnitude: every partial sum of a score stays far below 2^53
    rows, _, _ = lrc.graph(M, seed)
    deg = np.bincount(rows, minlength=M).max()
    assert deg <= 4
    assert lrc.score_bound(cfg["model"], r, deg) < 2.0 ** 43


def test_multirank_blocks_hold_padding_and_an_empty_rank():
    """The 1.5D A-row blocks of [k ceil(M/p), (k + 1) ceil(M/p)): at M = 301 the last rank holds padding rows, at M = 9
    and p = 4 the last rank holds none below M; the isolated copies sit on different ranks."""
    for p in (2, 4):
        b = lrc.block_rows(301, p)
        assert b[-1][1] < b[0][1] and sum(v for _, v in b) == 301
        owners = {int(i) // -(-301 // p) for i in lrc.isolated(301)}
        assert len(owners) >= 2
    assert lrc.block_rows(9, 4) == [(0, 3), (3, 3), (6, 3), (9, 0)]
    assert len({int(i) // 3 for i in lrc.isolated(9)}) >= 2
    # the wide multi-rank case crosses at least two chunk edges
    assert -(-(2 * 256 + 5) // lrc.chunk_of(65536)) == 3
