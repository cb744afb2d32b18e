"""fp64 torch models of filtered link ranking (include/hnh/link_ranking.hpp) -- TEST INFRASTRUCTURE.

`compute_mrr_loop` is PyG's examples/rgcn_link_pred.py (compute_rank / compute_mrr), literally: per query a Python loop
that builds the filter masks from the known triple sets and decodes [true, candidates...] with the DistMult decoder of
tests/distmult_oracle.py, in fp64 instead of the example's fp32.  `filtered_ranks` is the vectorised definition the
library implements: candidates exclude the true entity and F, rank = ((gt + 1) + (ge + 1)) / 2.  The two agree wherever
every query is in F; with the true triple missing from F the loop counts the true entity twice, so its rank is 0.5
higher.  Both associate the score as (z_u * rel) * z_v, summed by torch.  `matmul_ranks` is `filtered_ranks` by one
matrix product per query chunk with a vectorised filter mask: it scales to wide outputs and many queries, and on
integer-valued operands it is exact.  Nothing under distributed_sddmm_b200/ imports this module.
"""
from __future__ import annotations

import numpy as np
import torch

from tests.distmult_oracle import DistMultDecoder


def decoder_of(rel):
    """A distmult_oracle.DistMultDecoder whose rel_emb is rel (R x r); rel = ones((1, r)) is the dot product."""
    rel = torch.as_tensor(np.asarray(rel, np.float64))
    dec = DistMultDecoder(rel.shape[0], rel.shape[1])
    with torch.no_grad():
        dec.rel_emb.copy_(rel)
    return dec


@torch.no_grad()
def compute_rank(ranks):
    # fair ranking prediction as the average of optimistic and pessimistic ranking
    true = ranks[0]
    optimistic = (ranks > true).sum() + 1
    pessimistic = (ranks >= true).sum()
    return (optimistic + pessimistic).double() * 0.5


@torch.no_grad()
def compute_mrr_loop(z, model, queries, known, num_nodes):
    """PyG's compute_mrr: z (num_nodes x r), model the decoder, queries = (heads, rels, tails), known = a list of
    (heads, rels, tails) sets (the example's train, valid and test).  Returns (mrr, tail ranks, head ranks)."""
    z = torch.as_tensor(np.asarray(z, np.float64))
    src_all, rel_all, dst_all = (torch.as_tensor(np.asarray(a, np.int64)) for a in queries)
    known = [tuple(torch.as_tensor(np.asarray(a, np.int64)) for a in k) for k in known]
    tail_ranks, head_ranks = [], []
    for i in range(rel_all.numel()):
        src, dst, rel = src_all[i], dst_all[i], rel_all[i]

        # Try all nodes as tails, but delete true triplets:
        tail_mask = torch.ones(num_nodes, dtype=torch.bool)
        for heads, types, tails in known:
            tail_mask[tails[(heads == src) & (types == rel)]] = False
        tail = torch.arange(num_nodes)[tail_mask]
        tail = torch.cat([torch.tensor([dst]), tail])
        head = torch.full_like(tail, fill_value=src)
        eval_edge_index = torch.stack([head, tail], dim=0)
        eval_edge_type = torch.full_like(tail, fill_value=rel)
        out = model(z, eval_edge_index, eval_edge_type)
        tail_ranks.append(compute_rank(out))

        # Try all nodes as heads, but delete true triplets:
        head_mask = torch.ones(num_nodes, dtype=torch.bool)
        for heads, types, tails in known:
            head_mask[heads[(tails == dst) & (types == rel)]] = False
        head = torch.arange(num_nodes)[head_mask]
        head = torch.cat([torch.tensor([src]), head])
        tail = torch.full_like(head, fill_value=dst)
        eval_edge_index = torch.stack([head, tail], dim=0)
        eval_edge_type = torch.full_like(head, fill_value=rel)
        out = model(z, eval_edge_index, eval_edge_type)
        head_ranks.append(compute_rank(out))
    t, h = torch.stack(tail_ranks).numpy(), torch.stack(head_ranks).numpy()
    return float((1.0 / np.concatenate([t, h])).mean()), t, h


@torch.no_grad()
def filtered_ranks(z, rel, queries, known, num_nodes, chunk=256):
    """The library's definition, vectorised over query chunks: (mrr, tail ranks, head ranks, tail scores, head
    scores), the scores n_q x num_nodes (for checks that no decision is a rounding's)."""
    z = torch.as_tensor(np.asarray(z, np.float64))[:num_nodes]
    rel = torch.as_tensor(np.asarray(rel, np.float64))
    h, rho, t = (np.asarray(a, np.int64) for a in queries)
    F = np.concatenate([np.stack([np.asarray(a, np.int64) for a in k], 1) for k in known]) if known else np.zeros((0, 3), np.int64)
    R = rel.shape[0]
    key_tail = set(((F[:, 0] * R + F[:, 1]) * num_nodes + F[:, 2]).tolist())
    out_ranks, out_scores = [], []
    for tail in (True, False):
        ranks, scores = [], []
        for c0 in range(0, len(h), chunk):
            hh, rr, tt = (torch.as_tensor(a[c0:c0 + chunk]) for a in (h, rho, t))
            s = ((z[hh] * rel[rr])[:, None, :] * z[None, :, :]).sum(-1) if tail else \
                ((z[None, :, :] * rel[rr][:, None, :]) * z[tt][:, None, :]).sum(-1)  # n x num_nodes
            true = s[torch.arange(len(hh)), tt if tail else hh]
            cand = torch.ones_like(s, dtype=torch.bool)
            v = torch.arange(num_nodes)
            for q in range(len(hh)):
                if tail:
                    keys = (int(hh[q]) * R + int(rr[q])) * num_nodes + v
                else:
                    keys = (v * R + int(rr[q])) * num_nodes + int(tt[q])
                cand[q] = torch.as_tensor([k not in key_tail for k in keys.tolist()])
                cand[q, int(tt[q] if tail else hh[q])] = False
            gt = ((s > true[:, None]) & cand).sum(1)
            ge = ((s >= true[:, None]) & cand).sum(1)
            ranks.append(((gt + 1) + (ge + 1)).double() / 2)
            scores.append(s)
        out_ranks.append(torch.cat(ranks).numpy() if ranks else np.zeros(0))
        out_scores.append(torch.cat(scores).numpy() if scores else np.zeros((0, num_nodes)))
    allr = np.concatenate(out_ranks)
    mrr = float((1.0 / allr).mean()) if len(allr) else 0.0
    return mrr, out_ranks[0], out_ranks[1], out_scores[0], out_scores[1]


def separated(scores_t, scores_h, q):
    """True when every score either equals the true one or differs from it far beyond rounding (so that the
    oracle's association and the library's decide alike).  scores_t / scores_h are the n_q x num_nodes tail and head
    scores of filtered_ranks or matmul_ranks, q = (heads, rels, tails)."""
    for s, col in ((scores_t, q[2]), (scores_h, q[0])):
        true = s[np.arange(len(col)), col][:, None]
        d = np.abs(s - true)
        if not ((d == 0) | (d > 1e-9 * max(np.abs(s).max(), 1e-300))).all():
            return False
    return True


def filter_keys(known, R, num_nodes):
    """The sorted distinct int64 keys (h R + rho) num_nodes + t of the known triples."""
    if not known:
        return np.zeros(0, np.int64)
    F = np.concatenate([np.stack([np.asarray(a, np.int64) for a in k], 1) for k in known])
    return np.unique((F[:, 0] * R + F[:, 1]) * num_nodes + F[:, 2])


def matmul_ranks(z, rel, queries, known, num_nodes, chunk=None):
    """filtered_ranks by one matrix product per chunk of queries, (z[anchor] o rel[rho]) @ z.T, with the filter mask
    built by np.isin on int64 triple keys: the same tuple, at any width and any number of queries.  On integer-valued z
    and rel whose products and partial sums stay integers below 2^53 every score is exact whatever the summation order,
    so the ranks are the library's bit for bit with no separation guard."""
    z = np.ascontiguousarray(np.asarray(z, np.float64)[:num_nodes])
    rel = np.asarray(rel, np.float64)
    h, rho, t = (np.asarray(a, np.int64) for a in queries)
    R, n_q = rel.shape[0], len(h)
    chunk = chunk or max(1, (1 << 22) // max(z.shape[1], 1))  # a query block of at most 32 MB
    keys = filter_keys(known, R, num_nodes)
    v = np.arange(num_nodes, dtype=np.int64)
    out_ranks, out_scores = [], []
    for tail in (True, False):
        anchor, target = (h, t) if tail else (t, h)
        ranks, scores = np.zeros(n_q), np.zeros((n_q, num_nodes))
        for c0 in range(0, n_q, chunk):
            a, rr, tg = anchor[c0:c0 + chunk], rho[c0:c0 + chunk], target[c0:c0 + chunk]
            s = (z[a] * rel[rr]) @ z.T  # n x num_nodes
            true = s[np.arange(len(a)), tg]
            k = ((a * R + rr)[:, None] * num_nodes + v[None, :]) if tail else ((v[None, :] * R + rr[:, None]) * num_nodes + a[:, None])
            cand = ~np.isin(k, keys)
            cand[np.arange(len(a)), tg] = False
            gt = ((s > true[:, None]) & cand).sum(1)
            ge = ((s >= true[:, None]) & cand).sum(1)
            ranks[c0:c0 + chunk] = ((gt + 1) + (ge + 1)) / 2.0
            scores[c0:c0 + chunk] = s
        out_ranks.append(ranks)
        out_scores.append(scores)
    allr = np.concatenate(out_ranks)
    mrr = float((1.0 / allr).mean()) if len(allr) else 0.0
    return mrr, out_ranks[0], out_ranks[1], out_scores[0], out_scores[1]


def integer_bound(z, rel):
    """A bound on |any partial sum| of a score z_u . (z_v o rel_rho): r max|z|^2 max|rel|."""
    z, rel = np.asarray(z, np.float64), np.asarray(rel, np.float64)
    return float(z.shape[1]) * float(np.abs(z).max(initial=0.0)) ** 2 * float(np.abs(rel).max(initial=0.0))
