"""Multi-process worker for the multi-rank GraphSAGE tests (launched through torch.distributed.run by
tests/test_graph_sage_multirank_gpu.py).  Per case every rank builds S from its share of a global graph (its row slice
of an Erdos-Renyi graph, or its round-robin share of tests/skewed_graph.py's graph), then runs the case: the op
(Algorithm.max_aggregate and its backward), or GraphSAGE's forward and backward.  Results go to
<outdir>/<case>_rank<r>.npz, or the error every rank must raise."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import graph_sage_oracle as gso  # noqa: E402
from tests.mp_worker import gather_local  # noqa: E402
from tests.skewed_graph import rank_slice, skewed_tuples  # noqa: E402

LAYERS = [(8, 6), (6, 4)]


def global_graph(case):
    """(N, rows, cols) of the whole graph, the same on every rank."""
    from oracle import hnh_oracle as orc
    if case.get("skewed"):
        rows, cols = skewed_tuples(4200, 4200, case["seed"])
        return 4200, rows.astype(np.int64), cols.astype(np.int64)
    N = 1 << case["logM"]
    rows, cols, _ = orc.er_tuples(case["logM"], 5, case["seed"])
    return N, np.asarray(rows, np.int64), np.asarray(cols, np.int64)


def global_inputs(case, N):
    """(model params, X, G) for the model cases, (X, dZ) for the op: the same on every rank."""
    rng = np.random.default_rng(case["seed"] + 3)
    if case["model"] == "op":
        X = np.maximum(rng.standard_normal((N, case["f"])), 0.0)
        return X, rng.standard_normal((N, case["f"]))
    params = gso.random_params(LAYERS, rng)
    X = rng.uniform(-1, 1, (N, LAYERS[0][0]))
    G = rng.uniform(-1, 1, (N, LAYERS[-1][1]))
    return params, X, G


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
        name, alg_name, c = case["name"], case["alg"], case["c"]
        N, grows, gcols = global_graph(case)
        if case.get("skewed"):
            sr, sc_ = rank_slice(grows, gcols, rank, world)
        else:
            per = N // world
            sr, sc_, _ = orc.er_tuples(case["logM"], 5, case["seed"], per * rank, N if rank == world - 1 else per * (rank + 1))
        S = D.SpmatLocal.from_tuples(N, N, sr, sc_, np.ones(len(sr)))
        f0 = case["f"] if case["model"] == "op" else LAYERS[0][0]
        out = {}
        try:
            alg = D.Algorithm(alg_name, S, f0, c)
            topA, _, nrA, _ = alg.submatrices("A")[0]
            topB, _, nrB, _ = alg.submatrices("B")[0]
            out["topA"], out["topB"] = np.array([topA, nrA]), np.array([topB, nrB])
            if case["model"] == "op":
                X, dZh = global_inputs(case, N)
                f = case["f"]
                nA, nB = alg.like_A_matrix().shape[0], alg.like_B_matrix().shape[0]
                Xd, Z, Cn, dZ, dX = (D.Dense.create(n, f) for n in (nB, nA, nA, nA, nB))
                Xd.from_host(gather_local(X, [(topB, 0, nrB, f)], (nB, f)))
                dZ.from_host(gather_local(dZh, [(topA, 0, nrA, f)], (nA, f)))
                alg.max_aggregate(Xd, Z, Cn)
                alg.max_aggregate_backward(Xd, Z, Cn, dZ, dX)
                out["Z"], out["C"], out["dX"] = Z.to_host(), Cn.to_host(), dX.to_host()
                alg.max_aggregate(Xd, Z, Cn)
                alg.max_aggregate_backward(Xd, Z, Cn, dZ, dX)
                out["Z2"], out["dX2"] = Z.to_host(), dX.to_host()
            else:
                params, X, G = global_inputs(case, N)
                net = D.GraphSAGE(alg, LAYERS, aggr=case["aggr"])
                for l, P in enumerate(params):
                    for k, v in P.items():
                        net.set_param(l, k, v)
                net.set_input(gather_local(X, [(topB, 0, nrB, LAYERS[0][0])], net.buffer_shape(0)))
                net.forward()
                out["out"] = net.buffer(len(LAYERS))
                net.backward(gather_local(G, [(topA, 0, nrA, LAYERS[-1][1])], net.buffer_shape(len(LAYERS))))
                out["dX"] = net.input_grad()
                for l in range(len(LAYERS)):
                    for k in net.param_names():
                        out[f"g{l}_{k}"] = net.param_grad(l, k)
        except RuntimeError as e:
            out["error"] = str(e)
        np.savez(os.path.join(outdir, f"{name}_rank{rank}.npz"), **out)
        del S
    D.world_finalize()


if __name__ == "__main__":
    main()
