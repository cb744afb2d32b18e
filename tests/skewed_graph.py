"""A seeded skewed sparse pattern for the distributed tests -- TEST INFRASTRUCTURE (numpy only).

The Erdos-Renyi inputs of the other distributed tests have rows of at most a handful of entries, no empty stretch
and no hub.  skewed_tuples builds, by construction, what a real graph has and those lack.  With q = ceil(M / 4) and
w = ceil(N / 4), the row and column blocks of 4 ranks (landmarks(M, N) names all of this):

  * ordinary rows with power-law lengths (most 1 to 8 entries, a tail up to 400);
  * two wide hub rows (row 3 in the first row block, row q + 11 in the second) of more than 2 * 1024 + 37 distinct
    columns over the whole column range, more than 500 of them in each of the 4 column blocks, and a hub row (17)
    whose entries all lie in the last column block;
  * a hub column (7) that more than 60 % of the rows with entries point to;
  * more than 25 % rows without entries: the whole third row block [2 q, 3 q) and every row with row % 9 == 4;
    the rows of the last row block point to the first half of the columns only (and to nothing else, hubs aside), so
    the rank that owns them finds nothing in the other column blocks;
  * a band of ceil(N / 8) columns [w, w + ceil(N / 8)) that no entry touches (a whole column block of 8);
  * rows of exactly one entry, self-loops, and more than 50 duplicated (row, col) pairs, three of them in hub row 3
    (one of those stored three times).

The tuple list comes back shuffled (seeded), so no slice of it is aligned with ownership.
"""
from __future__ import annotations

import numpy as np

PIECE = 1024  # the edge softmax's piece length (kPiece in csrc/edge_softmax.cu)
HUB_MIN = 2 * PIECE + 37
DEFAULT_N = 4200
RECTANGULAR = [(2203, 4201), (5003, 4203)]  # M < N and M > N; none divisible by 4


def landmarks(M, N):
    """The fixed features of skewed_tuples(M, N, seed), for every seed."""
    q, w, e = -(-M // 4), -(-N // 4), -(-N // 8)
    return dict(q=q, w=w, wide_hubs=(3, q + 11), last_block_hub=17, hub_col=7, empty_rows=(2 * q, min(3 * q, M)),
                empty_cols=(w, w + e), narrow_rows=(3 * q, M), dup_row=3)


def skewed_tuples(M, N, seed, mean_tail=1.25, hub_share=0.65, hub_density=0.75, duplicates=60):
    """(rows, cols) as uint64: the global tuple list of an M x N pattern, in a fixed (shuffled) order."""
    rng = np.random.default_rng(seed)
    lm = landmarks(M, N)
    q, w = lm["q"], lm["w"]
    c0, c1 = lm["empty_cols"]
    free = np.concatenate([np.arange(0, c0), np.arange(c1, N)])  # the columns an entry may touch
    hubs = set(lm["wide_hubs"]) | {lm["last_block_hub"]}
    live = np.ones(M, bool)
    live[lm["empty_rows"][0]:lm["empty_rows"][1]] = False
    live[np.arange(M) % 9 == 4] = False
    live[list(hubs)] = True
    rr, cc = [], []
    # ordinary rows: power-law lengths
    ordinary = np.flatnonzero(live & ~np.isin(np.arange(M), list(hubs)))
    lens = np.minimum(np.floor(rng.pareto(mean_tail, len(ordinary)) * 3.0 + 1).astype(np.int64), 400)
    narrow = free[free < N // 2]
    for u, n in zip(ordinary, lens):
        pool = narrow if u >= lm["narrow_rows"][0] else free
        cols = rng.choice(pool, min(n, len(pool)), replace=False)
        rr.append(np.full(len(cols), u))
        cc.append(cols)
    # the hub column, skipping rows that would no longer have exactly one entry too often: a third of the one-entry rows
    # keep their single entry
    single = ordinary[lens == 1]
    to_hub = ordinary[rng.random(len(ordinary)) < hub_share + 0.1]
    to_hub = np.setdiff1d(to_hub, single[::3])
    rr.append(to_hub)
    cc.append(np.full(len(to_hub), lm["hub_col"]))
    # self-loops on every fifth ordinary row whose own column may be touched
    loops = ordinary[(ordinary % 5 == 0) & (ordinary < N) & (ordinary < lm["narrow_rows"][0])]
    loops = loops[np.isin(loops, free)]
    rr.append(loops)
    cc.append(loops)
    # wide hub rows: every free column of the block that holds the empty band, hub_density of the others
    for u in lm["wide_hubs"]:
        cols = free[(free // w == c0 // w) | (rng.random(len(free)) < hub_density)]
        rr.append(np.full(len(cols), u))
        cc.append(cols)
    last = free[free >= 3 * w]
    last = last[rng.random(len(last)) < 0.9]
    rr.append(np.full(len(last), lm["last_block_hub"]))
    cc.append(last)
    rows, cols = np.concatenate(rr), np.concatenate(cc)
    # one copy of every pair so far (the hub column and the self-loops may repeat a drawn entry)
    key = np.unique(rows * N + cols)
    rows, cols = key // N, key % N
    # duplicates: stored copies of existing pairs; three pairs of hub row dup_row, one of them twice
    pick = rng.choice(len(rows), duplicates, replace=False)
    in_hub = np.flatnonzero(rows == lm["dup_row"])
    hub_at = in_hub[[5, len(in_hub) // 3, len(in_hub) // 2, len(in_hub) // 2]]
    rows = np.concatenate([rows, rows[pick], rows[hub_at]])
    cols = np.concatenate([cols, cols[pick], cols[hub_at]])
    order = rng.permutation(len(rows))
    return rows[order].astype(np.uint64), cols[order].astype(np.uint64)


def rank_slice(rows, cols, rank, world):
    """The tuples rank `rank` of `world` hands to SpmatLocal.from_tuples: round-robin by index, which follows no
    ownership rule, so redistribution moves nearly all of them."""
    return rows[rank::world].copy(), cols[rank::world].copy()
