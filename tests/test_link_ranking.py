"""Filtered link ranking without a GPU: PyG's compute_mrr loop (tests/link_ranking_oracle.py) against the vectorised
definition the library implements, on small knowledge graphs with F = train + valid + test, the documented empty-F
difference, and the Hits@K helper of the Python results."""
import numpy as np
import pytest

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
