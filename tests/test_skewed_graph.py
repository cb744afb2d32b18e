"""The skewed-graph generator (tests/skewed_graph.py) has every feature the distributed tests rely on, for the default
and the rectangular sizes and three seeds, and is deterministic; and the per-entry fp64 models those tests compare
with count every stored copy of a duplicated pair, shown against dense masked models that add log(count) to a score.
No GPU."""
import numpy as np
import pytest

from tests import gat_softmax_oracle as gso
from tests import sparse_attention_oracle as sa
from tests.skewed_graph import DEFAULT_N, HUB_MIN, RECTANGULAR, landmarks, rank_slice, skewed_tuples


@pytest.mark.parametrize("seed", [1, 2, 0xC0FFEE + 211])
@pytest.mark.parametrize("M,N", [(DEFAULT_N, DEFAULT_N)] + RECTANGULAR)
def test_generator_has_every_feature(M, N, seed):
    rows, cols = skewed_tuples(M, N, seed)
    assert rows.dtype == np.uint64 and cols.dtype == np.uint64
    again = skewed_tuples(M, N, seed)
    assert np.array_equal(rows, again[0]) and np.array_equal(cols, again[1])
    other = skewed_tuples(M, N, seed + 1)
    assert len(other[0]) != len(rows) or not np.array_equal(other[0], rows)
    r, c = rows.astype(np.int64), cols.astype(np.int64)
    assert r.max() < M and c.max() < N and (M % 4 or M == DEFAULT_N) and 20000 < len(r) * DEFAULT_N / M < 60000
    lm = landmarks(M, N)
    q, w = lm["q"], lm["w"]
    lens = np.bincount(r, minlength=M)
    live = lens > 0
    # power-law lengths: most rows with entries hold 1 to 8, some hold more than 100
    assert (lens[live] <= 8).mean() > 0.7 and (lens[live] > 100).sum() > 10 and np.median(lens[live]) <= 5
    # wide hub rows: more than two softmax pieces of distinct columns, more than 500 in each of 4 column blocks
    for u in lm["wide_hubs"]:
        cu = np.unique(c[r == u])
        assert len(cu) >= 2100 > HUB_MIN and all(((cu // w) == b).sum() > 500 for b in range(4)), (u, len(cu))
    assert lm["wide_hubs"][0] < q <= lm["wide_hubs"][1] < 2 * q  # in two different row blocks
    last = c[r == lm["last_block_hub"]]
    assert len(last) > 500 and last.min() >= 3 * w
    # the hub column
    assert len(np.unique(r[c == lm["hub_col"]])) > 0.6 * live.sum()
    # empty rows: more than a quarter, a whole row block of 4 among them; a column band nothing touches; the last row
    # block points to the first half of the columns only
    assert (~live).mean() > 0.25 and not live[lm["empty_rows"][0]:lm["empty_rows"][1]].any()
    assert lm["empty_rows"] == (2 * q, min(3 * q, M))
    touched = np.bincount(c, minlength=N) > 0
    e0, e1 = lm["empty_cols"]
    assert not touched[e0:e1].any() and e1 - e0 == -(-N // 8) and e0 == w
    assert c[r >= lm["narrow_rows"][0]].max() < N // 2 and live[lm["narrow_rows"][0]:].any()
    # one-entry rows, self-loops, duplicates (some in a hub row, one pair stored three times)
    assert (lens == 1).sum() > 50 and (r == c).sum() > 50
    key, count = np.unique(r * N + c, return_counts=True)
    assert (count > 1).sum() >= 50 and count.max() == 3
    assert (count[key // N == lm["dup_row"]] > 1).sum() >= 3
    # the shares handed to the ranks: round-robin, a partition, not aligned with row ownership
    for world in (2, 4):
        parts = [rank_slice(rows, cols, k, world) for k in range(world)]
        assert sum(len(p[0]) for p in parts) == len(rows)
        assert np.array_equal(np.sort(np.concatenate([p[0] * np.uint64(N) + p[1] for p in parts])), np.sort(rows * np.uint64(N) + cols))
        own = parts[0][0].astype(np.int64) // -(-M // world)
        assert (own != 0).mean() > 0.2  # rank 0 is handed tuples of rows it does not own


def _small():
    N = 300
    r, c = (x.astype(np.int64) for x in skewed_tuples(N, N, 7))
    order = np.lexsort((c, r))
    r, c = r[order], c[order]
    assert (np.diff(r * N + c) == 0).sum() >= 50
    return N, r, c


def test_attention_model_counts_every_copy_of_a_duplicate():
    N, r, c = _small()
    rng = np.random.default_rng(3)
    Q, K, V = (rng.uniform(-1, 1, (N, 16)) for _ in range(3))
    Z, L = sa.forward_np(r, c, N, Q, K, V, 2, 0.35)
    want = sa.dense_masked_np(r, c, N, N, Q, K, V, 2, 0.35)
    assert np.abs(Z - want).max() < 1e-13
    # and merging the copies would be seen: the model on the de-duplicated pattern differs
    key = np.unique(r * N + c)
    Zu, _ = sa.forward_np(key // N, key % N, N, Q, K, V, 2, 0.35)
    assert np.abs(Zu - want).max() > 1e-3
    assert np.isneginf(L[np.bincount(r, minlength=N) == 0]).all()


def test_edge_softmax_model_counts_every_copy_of_a_duplicate():
    N, r, c = _small()
    x = np.sin(0.37 * r + 1.91 * c) * 5
    alpha = gso.edge_softmax_np(x, r, N)
    count = np.zeros((N, N))
    np.add.at(count, (r, c), 1.0)
    dense = np.full((N, N), -np.inf)
    dense[r, c] = x
    with np.errstate(divide="ignore", invalid="ignore"):
        e = np.exp(dense - np.nanmax(np.where(count > 0, dense, -np.inf), 1, keepdims=True) + np.log(count))
    e[count == 0] = 0
    s = e.sum(1, keepdims=True)
    want = (e / np.where(s > 0, s, 1) / np.where(count > 0, count, 1))[r, c]  # each copy gets its share of the pair's weight
    assert np.abs(alpha - want).max() < 1e-14
    sums = np.zeros(N)
    np.add.at(sums, r, alpha)
    assert np.abs(sums[np.bincount(r, minlength=N) > 0] - 1).max() < 1e-13
