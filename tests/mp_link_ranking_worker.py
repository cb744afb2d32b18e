"""Multi-process worker for the multi-rank filtered link-ranking tests (launched through torch.distributed.run by
tests/test_link_ranking_multirank_gpu.py).  Per case every rank builds the model's S from its row slice of an
Erdos-Renyi graph with hashed relations, sets the same R-GCN parameters, input and DistMult relation table, builds the
same filter and runs net.link_rank on the same queries -- or, for a refusal case, queries changed on one rank only.
Results go to <outdir>/<case>_rank<r>.npz: the ranks, the MRR and this rank's output rows; or the error."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

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
        name, alg_name, c, logM, seed = (case[k] for k in ("name", "alg", "c", "logM", "seed"))
        N = 1 << logM
        per = N // world
        sr, sc_, _ = orc.er_tuples(logM, 5, seed + 1, per * rank, N if rank == world - 1 else per * (rank + 1))
        sr, sc_ = np.asarray(sr, np.int64), np.asarray(sc_, np.int64)
        keep = ~np.isin(sr, isolated(N))
        sr, sc_ = sr[keep], sc_[keep]
        out = {}
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
