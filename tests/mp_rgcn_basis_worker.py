"""Multi-process worker for the multi-rank tests of R-GCN with basis decomposition (launched through torch.distributed.run
by tests/test_rgcn_basis_multirank_gpu.py).  Per case every rank builds S from its share of a global graph (its row slice
of an Erdos-Renyi graph, or its round-robin share of tests/skewed_graph.py's graph) with each entry's relation as its
value, then runs the case: the op (Algorithm.basis_aggregate and its backward, with the mean's scale), or the basis
RGCN's forward and backward and three train steps.  Results go to <outdir>/<case>_rank<r>.npz, or the error every rank
must raise."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import rgcn_basis_oracle as bo  # noqa: E402
from tests.mp_rgcn_worker import R, er_relations  # noqa: E402
from tests.mp_worker import gather_local  # noqa: E402
from tests.skewed_graph import rank_slice, skewed_tuples  # noqa: E402

LAYERS = [(8, 6), (6, 4)]
B = 3


def global_graph(case):
    """(N, rows, cols, rels) of the whole graph, the same on every rank."""
    from oracle import hnh_oracle as orc
    if case.get("skewed"):
        rows, cols = skewed_tuples(4200, 4200, case["seed"])
        rows, cols = rows.astype(np.int64), cols.astype(np.int64)
        return 4200, rows, cols, bo.ro.hashed_relations(rows, cols, 4200, R)
    N = 1 << case["logM"]
    rows, cols, _ = orc.er_tuples(case["logM"], 5, case["seed"])
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    return N, rows, cols, er_relations(rows, cols)


def global_inputs(case, N):
    """(model params, X, G) for the model cases, (X, dH, comp) for the op: the same on every rank."""
    rng = np.random.default_rng(case["seed"] + 3)
    if case["model"] == "op":
        return rng.standard_normal((N, case["f"])), rng.standard_normal((N, B * case["f"])), rng.standard_normal((R, B))
    params = bo.random_params(LAYERS, R, B, rng)
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
        N, grows, gcols, grels = global_graph(case)
        if case.get("skewed"):
            sr, sc_ = rank_slice(grows, gcols, rank, world)
            sv = grels[rank::world].copy()
        else:
            per = N // world
            sr, sc_, _ = orc.er_tuples(case["logM"], 5, case["seed"], per * rank, N if rank == world - 1 else per * (rank + 1))
            sv = er_relations(sr, sc_)
        S = D.SpmatLocal.from_tuples(N, N, sr, sc_, sv)
        f0 = case["f"] if case["model"] == "op" else LAYERS[0][0]
        out = {}
        try:
            alg = D.Algorithm(alg_name, S, f0, c)
            topA, _, nrA, _ = alg.submatrices("A")[0]
            topB, _, nrB, _ = alg.submatrices("B")[0]
            out["topA"], out["topB"] = np.array([topA, nrA]), np.array([topB, nrB])
            if case["model"] == "op":
                X, dHh, comp = global_inputs(case, N)
                f = case["f"]
                nA, nB = alg.like_A_matrix().shape[0], alg.like_B_matrix().shape[0]
                Xd, H, dH, dX = D.Dense.create(nB, f), D.Dense.create(nA, B * f), D.Dense.create(nA, B * f), D.Dense.create(nB, f)
                scale = D.Dense.create(nA, R)
                Xd.from_host(gather_local(X, [(topB, 0, nrB, f)], (nB, f)))
                dH.from_host(gather_local(dHh, [(topA, 0, nrA, B * f)], (nA, B * f)))
                scale.from_host(gather_local(bo.mean_scale(grows, grels, N, R), [(topA, 0, nrA, R)], (nA, R)))
                alg.basis_aggregate(Xd, H, comp, R, scale)
                out["dcomp"] = alg.basis_aggregate_backward(dH, Xd, dX, comp, R, scale)
                out["H"], out["dX"] = H.to_host(), dX.to_host()
                alg.basis_aggregate(Xd, H, comp, R, scale)
                out["dcomp2"] = alg.basis_aggregate_backward(dH, Xd, dX, comp, R, scale)
                out["H2"], out["dX2"] = H.to_host(), dX.to_host()
            else:
                params, X, G = global_inputs(case, N)
                net = D.RGCN(alg, LAYERS, num_relations=R, aggr=case["aggr"], num_bases=B)
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
                lab = np.full(net.buffer_shape(len(LAYERS))[0], -1)
                rows_here = min(nrA, max(N - topA, 0))
                lab[:rows_here] = (np.arange(topA, topA + rows_here) * 5) % LAYERS[-1][1]
                labels = D.NodeLabels(net, lab, LAYERS[-1][1])
                opt = D.AdamW(lr=1e-2)
                for _ in range(3):
                    net.train_step(labels, opt)
                for l in range(len(LAYERS)):
                    for k in net.param_names():
                        out[f"t{l}_{k}"] = net.param(l, k)
        except RuntimeError as e:
            out["error"] = str(e)
        np.savez(os.path.join(outdir, f"{name}_rank{rank}.npz"), **out)
        del S
    D.world_finalize()


if __name__ == "__main__":
    main()
