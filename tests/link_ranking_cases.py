"""Integer-valued link-ranking fixtures -- TEST INFRASTRUCTURE, no GPU.

GraphSAGE with aggr="sum", GIN with eps = 0 and R-GCN with aggr="sum" (with and without bases) give exact integer
outputs when their input, parameters and graph weights are small integers: every aggregation weight is 1, ReLU keeps
integers and the fp64 GEMMs are exact on them.  With an integer DistMult relation table every score and partial sum
is an integer far below 2^53, so tests/link_ranking_oracle.matmul_ranks gives the library's ranks bit for bit.  The
cases below make the last layer wide, so that link_rank splits the queries into several chunks of
chunk_of(r) = max(64, floor(kRankChunkDoubles / r / 64) 64) (include/hnh/link_ranking.hpp), and place the queries at
the chunk edges: a query repeated at positions k chunk - 1 and k chunk, self-loops, a hub (head, relation) whose
filter holds every node, a (head, relation) with no known triple, and targets that are copies of one output row
(isolated nodes with one input row, in different 64-row tiles and, at p > 1, on different ranks).
"""
from __future__ import annotations

import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F_IN = 4  # input width
HIDDEN = 8  # the hidden width of the two-layer models and of GIN's MLP


def rank_chunk_doubles():
    """kRankChunkDoubles, read from include/hnh/link_ranking.hpp."""
    with open(os.path.join(ROOT, "include", "hnh", "link_ranking.hpp")) as f:
        m = re.search(r"constexpr int64_t kRankChunkDoubles = int64_t\(1\) << (\d+);", f.read())
    assert m, "kRankChunkDoubles not found"
    return 1 << int(m.group(1))


def chunk_of(r, n_q=None):
    """The queries per chunk linkRank uses at output width r (n_q caps it)."""
    c = max(64, rank_chunk_doubles() // r // 64 * 64)
    return c if n_q is None else min(n_q, c)


def block_rows(M, p):
    """The 1.5D layouts' A-row block of each rank: [k ceil(M/p), (k + 1) ceil(M/p)); returns (top, valid) per rank."""
    per = -(-M // p)
    return [(k * per, max(0, min(per, M - k * per))) for k in range(p)]


def isolated(M):
    """Nodes without S entries and with one input row: their output rows are copies.  At M >= 201 they sit in five
    different 64-row tiles; at least three of them at any M >= 5."""
    iso = {x for x in (3, 70, 140, 200, M - 1) if x < M}
    return np.array(sorted(iso if len(iso) >= 3 else iso | {M // 2}), np.int64)


# name -> model, output width r, M, decoder relations (None: dot product), queries
WIDE = {
    "sage_r65536_dot": dict(model="sage", r=65536, M=300, R=None, n_q=257),  # one more than one chunk
    "rgcn_r40001_distmult": dict(model="rgcn", r=40001, M=200, R=3, n_q=2 * 384 + 100),  # two chunks and a partial
    "rgcn_bases_r65536_distmult": dict(model="rgcn_bases", r=65536, M=300, R=3, n_q=256),  # exactly one chunk
    "gin_r262145_dot": dict(model="gin", r=262145, M=40, R=None, n_q=2 * 64 + 23),  # the 64-query floor
    "sage_r262145_distmult": dict(model="sage", r=262145, M=40, R=3, n_q=64 + 1),
}
# what each case's chunk must reach: (chunk, number of chunks, last chunk partial)
WIDE_REACHES = {
    "sage_r65536_dot": (256, 2, True),
    "rgcn_r40001_distmult": (384, 3, True),
    "rgcn_bases_r65536_distmult": (256, 1, False),
    "gin_r262145_dot": (64, 3, True),
    "sage_r262145_distmult": (64, 2, True),
}
RELS = 3  # R-GCN's relation count (the relations of S's entries)
BASES = 2  # R-GCN's basis count with bases
ZERO_REL, UNUSED_REL = 1, 2  # with a decoder of 3 relations: an all-zero relation row, and one no query uses


def case_seed(name):
    """The seed of the wide case `name`: its graph, parameters, input and relation table draw from case_seed .. + 3,
    its filter and queries from case_seed + 4."""
    return 0xC0FFEE + 493 + len(name)


def score_bound(model, r, deg):
    """A bound on |every partial sum of a score| of `model` r wide with the parameters of integer_param (not nonneg),
    |X| <= 1, at most deg entries per S-row and a relation table of integer_param's range (|D| <= 2).  max |W| is 1
    for every weight, except R-GCN with bases, whose W_rho = sum_b comp[rho, b] V_b reaches BASES.  Sum aggregation
    over deg entries and the root term give (deg + 1) |X| max|W| per input feature; R-GCN's relations split those deg
    entries, so they add no factor."""
    w = BASES if model == "rgcn_bases" else 1
    bias = 2
    if model == "gin":  # H = sum + X, then Linear(F_IN, HIDDEN), ReLU, Linear(HIDDEN, r)
        hidden = (deg + 1) * F_IN * w + bias
        out = HIDDEN * hidden * w + bias
    else:  # two layers: F_IN -> HIDDEN (ReLU) -> r
        hidden = (deg + 1) * F_IN * w + bias
        out = (deg + 1) * HIDDEN * hidden * w + bias
    return r * out * out * 2


def graph(M, seed, per_row=4):
    """(rows, cols, relations) of S: per_row entries per row (some may repeat), none in the isolated nodes' rows,
    relations in [0, 3)."""
    rng = np.random.default_rng(seed)
    rows = np.repeat(np.arange(M, dtype=np.int64), per_row)
    cols = rng.integers(0, M, len(rows)).astype(np.int64)
    keep = ~np.isin(rows, isolated(M))
    rows, cols = rows[keep], cols[keep]
    return rows, cols, ((rows * 7 + cols * 3) % RELS).astype(np.float64)


def layers(model, r):
    if model == "gin":
        return [(F_IN, HIDDEN, r)]
    return [(F_IN, HIDDEN), (HIDDEN, r)]


def integer_input(M, seed, nonneg=False):
    """M x F_IN small integers; the isolated nodes share one row."""
    rng = np.random.default_rng(seed)
    X = rng.integers(0 if nonneg else -1, 3 if nonneg else 2, (M, F_IN)).astype(np.float64)
    X[isolated(M)] = X[isolated(M)[0]]
    return X


def integer_param(shape, rng, nonneg=False):
    """Weights (2-D, and R-GCN's basis coefficients) in {-1, 0, 1} ({0, 1} with nonneg), vectors (biases) in [-2, 2]
    ([0, 2])."""
    if len(shape) == 1:
        return rng.integers(0 if nonneg else -2, 3, shape).astype(np.float64)
    return rng.integers(0 if nonneg else -1, 2, shape).astype(np.float64)


def relation_table(R, r, seed, nonneg=False):
    """R x r integers in [-2, 2] ([0, 2]), row ZERO_REL all zero (every candidate ties)."""
    rng = np.random.default_rng(seed)
    D = rng.integers(0 if nonneg else -2, 3, (R, r)).astype(np.float64)
    D[ZERO_REL] = 0.0
    return D


def queries(M, R, n_q, chunk, seed):
    """(filter triples, queries, lonely, hub, chunk edges).  The filter: random triples and the first half of the
    queries, none touching the node `lonely`, and every (hub, 0, v).  The queries: random ones on the relations other
    than UNUSED_REL; a tie query repeated at positions k chunk - 1 and k chunk; self-loops; hub queries (tail rank 1);
    queries with an empty tail filter (lonely, 0, t) and with the hub alone as head filter (h, 0, lonely); queries
    whose true tail or head is an isolated node, whose copies tie with it; with a decoder, all-zero relation queries."""
    rng = np.random.default_rng(seed)
    iso = isolated(M)
    hub, lonely = 1 % M, M - 2
    others = np.setdiff1d(np.arange(M), [lonely])
    used = [0] if R == 1 else [0, ZERO_REL]
    h, rho, t = rng.choice(others, n_q), rng.choice(used, n_q), rng.choice(others, n_q)
    special = [(5 % M, 0, 5 % M), (iso[0], 0, iso[0]), (hub, 0, 7 % M), (hub, 0, iso[1]), (lonely, 0, 9 % M),
               (11 % M, 0, lonely), (13 % M, 0, iso[-1]), (iso[-1], 0, 15 % M), (iso[1], 0, iso[0])]
    if R > 1:
        special += [(17 % M, ZERO_REL, 19 % M), (hub, ZERO_REL, iso[0])]
    edges = [k * chunk for k in range(1, -(-n_q // chunk)) if k * chunk < n_q]
    taken = set(edges) | {e - 1 for e in edges}
    free = [i for i in range(n_q) if i not in taken]
    for i, s in zip(free[::max(1, len(free) // len(special))], special):
        h[i], rho[i], t[i] = s
    for k, e in enumerate(edges):  # a tie query (an isolated target) on both sides of every chunk edge
        h[e - 1], rho[e - 1], t[e - 1] = (21 + k) % M, used[k % len(used)], iso[k % len(iso)]
        h[e], rho[e], t[e] = h[e - 1], rho[e - 1], t[e - 1]
    q = (h.astype(np.int64), rho.astype(np.int64), t.astype(np.int64))
    fh, fr, ft = rng.choice(others, 6 * M), rng.integers(0, R, 6 * M), rng.choice(others, 6 * M)
    F = (np.concatenate([fh, q[0][:n_q // 2]]), np.concatenate([fr, q[1][:n_q // 2]]), np.concatenate([ft, q[2][:n_q // 2]]))
    keep = (F[0] != lonely) & (F[2] != lonely)
    F = (np.concatenate([F[0][keep], np.full(M, hub)]), np.concatenate([F[1][keep], np.zeros(M, np.int64)]),
         np.concatenate([F[2][keep], np.arange(M)]))
    return tuple(a.astype(np.int64) for a in F), q, lonely, hub, edges
