"""Multi-process worker for the multi-rank filtered link-ranking tests (launched through torch.distributed.run by
tests/test_link_ranking_multirank_gpu.py).  Per case every rank builds the model's S from its row slice of an
Erdos-Renyi graph with hashed relations, sets the same R-GCN parameters, input and DistMult relation table, builds the
same filter and runs net.link_rank on the same queries -- or, for a refusal case, queries changed on one rank only.
Results go to <outdir>/<case>_rank<r>.npz: the ranks, the MRR and this rank's output rows; or the error.

A case with "model" ranks another model on M nodes (any M; every rank takes a strided slice of one global tuple list):
"sage_wide", a one-layer GraphSAGE (sum) r wide with non-negative integer parameters and a non-negative integer
DistMult table (tests/link_ranking_cases.py), whose scores are exact; "gat" (softmax attention) and "gine", float
models ranked by dot product.  "pad" is written into every padding row (global row >= M) of each rank's input: GraphSAGE
maps it to output rows that outscore every true entity, so a rank that counted them would differ."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import gin_oracle as go  # noqa: E402
from tests import link_ranking_cases as lrc  # noqa: E402
from tests import rgcn_oracle as ro  # noqa: E402
from tests.mp_worker import gather_local  # noqa: E402

LAYERS = [(8, 12), (12, 8)]
R = 4


def s_relations(rows, cols):
    return ((rows * 7 + cols * 3) % R).astype(np.float64)


def global_inputs(case):
    """(filter triples, queries, model params, X, rel), the same on every rank.  The nodes 1, 2 and N - 2 have no
    entries and one input row, so their output rows are copies (on different ranks at p > 1)."""
    N = 1 << case["logM"]
    rng = np.random.default_rng(case["seed"])
    h, rr, t = rng.integers(0, N, 6 * N), rng.integers(0, R, 6 * N), rng.integers(0, N, 6 * N)
    hub = N // 2 + 10
    h[:hub], rr[:hub], t[:hub] = 5, 1, rng.permutation(N)[:hub]  # a hub (head, relation): more than half the nodes known
    F = (h.astype(np.int64), rr.astype(np.int64), t.astype(np.int64))
    pick = rng.choice(len(h), 120, replace=False)
    q = tuple(np.concatenate([a[pick], a[pick[:6]]]) for a in F)  # every query is known; 6 duplicates
    q = (np.concatenate([q[0], [3, 1]]), np.concatenate([q[1], [0, 2]]), np.concatenate([q[2], [2, 9]]))
    F = tuple(np.concatenate([a, b[-2:]]) for a, b in zip(F, q))
    params = ro.random_params(LAYERS, R, rng)
    X = rng.uniform(-1, 1, (N, LAYERS[0][0]))
    X[[2, N - 2]] = X[1]
    rel = rng.uniform(-1, 1, (R, LAYERS[-1][1]))
    return F, q, params, X, rel


def isolated(N):
    return np.array([1, 2, N - 2])


WIDE_R = 3  # the DistMult relations of the "sage_wide" cases


def model_layers(case):
    return {"sage_wide": [(lrc.F_IN, case.get("r", 0))], "gat": [(lrc.F_IN, 4, 2), (8, 6, 1)],
            "gine": [(lrc.F_IN, 8, 6)]}[case["model"]]


def model_inputs(case):
    """(S tuples (rows, cols), filter triples, queries, params [per layer {name: array}], X, rel or None), the same
    on every rank, for a case with a "model"."""
    M, r, seed = case["M"], case.get("r", 0), case["seed"]
    rows, cols, _ = lrc.graph(M, seed)
    rng = np.random.default_rng(seed + 1)
    layers = model_layers(case)
    if case["model"] == "sage_wide":
        f = lrc.F_IN
        P = {"neigh": lrc.integer_param((f, r), rng, True), "neigh_bias": lrc.integer_param((r,), rng, True),
             "root": lrc.integer_param((f, r), rng, True)}
        P["root"][np.arange(r) % f, np.arange(r)] = 1.0  # a padding row of value L scores >= L in every column
        n_q = case["n_q"]
        F, q, _, _, _ = lrc.queries(M, WIDE_R, n_q, lrc.chunk_of(r, n_q), seed + 4)
        return (rows, cols), F, q, [P], lrc.integer_input(M, seed + 2, True), lrc.relation_table(WIDE_R, r, seed + 3, True)
    if case["model"] == "gat":
        params = [{"weight": [rng.uniform(-1, 1, (fi, d)) / np.sqrt(fi) for _ in range(H)],
                   "a": [(rng.uniform(-1, 1, d), rng.uniform(-1, 1, d)) for _ in range(H)]} for fi, d, H in layers]
    else:
        params = go.random_params(layers, 3, rng)
    F = (rng.integers(0, M, 4 * M), np.zeros(4 * M, np.int64), rng.integers(0, M, 4 * M))
    q = tuple(np.concatenate([a[:60], b]) for a, b in zip(F, (rng.integers(0, M, 60), np.zeros(60, np.int64), rng.integers(0, M, 60))))
    return (rows, cols), F, q, params, rng.uniform(-1, 1, (M, lrc.F_IN)), None


def model_case(case, rank, world, alg_name, c):
    """(net, decoder or None, ranking, queries) of a case with a "model" on this rank."""
    from distributed_sddmm_b200 import driver as D
    M = case["M"]
    (rows, cols), F, q, params, X, rel = model_inputs(case)
    rows, cols = rows[rank::world], cols[rank::world]
    layers = model_layers(case)
    alg = D.Algorithm(alg_name, D.SpmatLocal.from_tuples(M, M, rows, cols, np.ones(len(rows))), lrc.F_IN, c)
    if case["model"] == "gat":
        net = D.GAT(alg, layers, attention="softmax")
        for l, P in enumerate(params):
            for h, (w, (a1, a2)) in enumerate(zip(P["weight"], P["a"])):
                net.set_weight(l, h, w)
                net.set_attention_vectors(l, h, a1, a2)
    else:
        net = D.GraphSAGE(alg, layers, aggr="sum") if case["model"] == "sage_wide" else D.GIN(alg, layers, edge_dim=3, eps=0.25)
        for l, P in enumerate(params):
            for k, v in P.items():
                if k != "eps":  # GINE keeps its constructor's eps
                    net.set_param(l, k, v)
        if case["model"] == "gine":
            net.set_edge_attributes(go.attr_of(*alg.entry_coordinates("A"), 3), go.attr_of(*alg.entry_coordinates("B"), 3))
    topB, _, nrB, _ = alg.submatrices("B")[0]
    Xl = gather_local(X, [(topB, 0, nrB, lrc.F_IN)], net.buffer_shape(0))
    Xl[max(0, M - topB):nrB] = case.get("pad", 0.0)  # the padding rows
    net.set_input(Xl)
    dec = None
    if rel is not None:
        dec = D.DistMultDecoder(net, len(rel))
        dec.set_param("rel", rel)
    return net, dec, D.LinkRanking(net, F, 1 if rel is None else len(rel)), q, alg


def main():
    cases = json.loads(sys.argv[1])
    outdir = sys.argv[2]
    transport = sys.argv[3]
    import torch
    ngpu = torch.cuda.device_count()
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")) % ngpu if transport == "nccl" else 0)
    from distributed_sddmm_b200 import driver as D
    from oracle import hnh_oracle as orc
    rank, world = D.world_init(transport)

    for case in cases:
        name, alg_name, c = (case[k] for k in ("name", "alg", "c"))
        out = {}
        if case.get("model"):
            try:
                net, dec, ranking, q, alg = model_case(case, rank, world, alg_name, c)
                res = net.link_rank(ranking, q, decoder=dec)
                again = net.link_rank(ranking, q, decoder=dec)
                out["tail"], out["head"], out["mrr"] = res.tail_ranks, res.head_ranks, np.array([res.mrr])
                out["again"] = np.concatenate([again.tail_ranks, again.head_ranks, [again.mrr]])
                topA, _, nrA, _ = alg.submatrices("A")[0]
                out["z"], out["top"] = net.buffer(len(net.layers)), np.array([topA])
            except RuntimeError as e:
                out["error"] = str(e)
            np.savez(os.path.join(outdir, f"{name}_rank{rank}.npz"), **out)
            continue
        logM, seed = case["logM"], case["seed"]
        N = 1 << logM
        per = N // world
        sr, sc_, _ = orc.er_tuples(logM, 5, seed + 1, per * rank, N if rank == world - 1 else per * (rank + 1))
        sr, sc_ = np.asarray(sr, np.int64), np.asarray(sc_, np.int64)
        keep = ~np.isin(sr, isolated(N))
        sr, sc_ = sr[keep], sc_[keep]
        try:
            alg = D.Algorithm(alg_name, D.SpmatLocal.from_tuples(N, N, sr, sc_, s_relations(sr, sc_)), LAYERS[0][0], c)
            F, q, params, X, rel = global_inputs(case)
            if case.get("bad") and case.get("bad_rank") == rank:
                q = tuple(a.copy() for a in q)
                q[2][7] = N if case["bad"] == "id" else (q[2][7] + 1) % N
            net = D.RGCN(alg, LAYERS, num_relations=R)
            for l, P in enumerate(params):
                for k, v in P.items():
                    net.set_param(l, k, v)
            topB, _, nrB, _ = alg.submatrices("B")[0]
            net.set_input(gather_local(X, [(topB, 0, nrB, LAYERS[0][0])], net.buffer_shape(0)))
            dec = D.DistMultDecoder(net, R)
            dec.set_param("rel", rel)
            ranking = D.LinkRanking(net, F, R)
            res = net.link_rank(ranking, q, decoder=dec)
            again = net.link_rank(ranking, q, decoder=dec)
            out["tail"], out["head"], out["mrr"] = res.tail_ranks, res.head_ranks, np.array([res.mrr])
            out["again"] = np.concatenate([again.tail_ranks, again.head_ranks, [again.mrr]])
            topA, _, nrA, _ = alg.submatrices("A")[0]
            out["z"], out["top"] = net.buffer(len(LAYERS)), np.array([topA])
        except RuntimeError as e:
            out["error"] = str(e)
        np.savez(os.path.join(outdir, f"{name}_rank{rank}.npz"), **out)
    D.world_finalize()


if __name__ == "__main__":
    main()
