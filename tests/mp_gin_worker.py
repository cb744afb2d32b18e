"""Multi-process worker for the multi-rank GIN tests (launched through torch.distributed.run by
tests/test_gin_multirank_gpu.py).  Per case every rank builds S from its row slice of a global Erdos-Renyi graph, then
runs the case: the op (Algorithm.edge_relu_aggregate and its backward), GIN's / GINE's forward and backward, or their
node train steps.  Results go to <outdir>/<case>_rank<r>.npz, or the error the rank raised."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import gin_oracle as go  # noqa: E402
from tests.mp_worker import gather_local  # noqa: E402

LAYERS = [(8, 10, 6), (6, 7, 4)]
CLASSES = 4


def global_graph(case):
    """(N, rows, cols) of the whole graph, the same on every rank."""
    from oracle import hnh_oracle as orc
    N = 1 << case["logM"]
    rows, cols, _ = orc.er_tuples(case["logM"], 5, case["seed"])
    return N, np.asarray(rows, np.int64), np.asarray(cols, np.int64)


def global_inputs(case, N):
    """(X, dA) for the op -- integer X, so that X_v + E_i == 0 happens -- and (params, X, G, labels) for the model: the
    same on every rank."""
    rng = np.random.default_rng(case["seed"] + 3)
    if case["model"] == "op":
        f = case["f"]
        return rng.integers(-2, 3, (N, f)).astype(np.float64), rng.standard_normal((N, f))
    params = go.random_params(LAYERS, case["edge_dim"], rng)
    X = rng.uniform(-1, 1, (N, LAYERS[0][0]))
    G = rng.uniform(-1, 1, (N, LAYERS[-1][2]))
    labels = rng.integers(0, CLASSES, N)
    labels[rng.random(N) < 0.3] = -1
    return params, X, G, labels


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
        N, _, _ = global_graph(case)
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
                X, dAh = global_inputs(case, N)
                f = case["f"]
                nA, nB = alg.like_A_matrix().shape[0], alg.like_B_matrix().shape[0]
                Xd, A, dA, dX, dE = (D.Dense.create(nB, f), D.Dense.create(nA, f), D.Dense.create(nA, f), D.Dense.create(nB, f),
                                     D.Dense.create(0, 0))
                ra, ca = alg.entry_coordinates("A")
                rb, cb = alg.entry_coordinates("B")
                EA, EB = D.Dense.create(len(ra), f), D.Dense.create(len(rb), f)
                if len(ra):
                    EA.from_host(go.edge_rows(ra, ca, f))
                if len(rb):
                    EB.from_host(go.edge_rows(rb, cb, f))
                Xd.from_host(gather_local(X, [(topB, 0, nrB, f)], (nB, f)))
                dA.from_host(gather_local(dAh, [(topA, 0, nrA, f)], (nA, f)))
                out["ra"], out["ca"] = ra, ca
                for k in ("", "2"):  # twice: repeats are bit-identical
                    alg.edge_relu_aggregate(Xd, EA, A)
                    alg.edge_relu_aggregate_backward(Xd, EA, EB, dA, dX, dE)
                    out["A" + k], out["dX" + k], out["dE" + k] = A.to_host(), dX.to_host(), dE.to_host()
            else:
                params, X, G, labels = global_inputs(case, N)
                e = case["edge_dim"]
                net = D.GIN(alg, LAYERS, edge_dim=e, eps=0.5, train_eps=True)
                for l, P in enumerate(params):
                    for k, v in P.items():
                        net.set_param(l, k, v)
                if e:
                    net.set_edge_attributes(go.attr_of(*alg.entry_coordinates("A"), e), go.attr_of(*alg.entry_coordinates("B"), e))
                net.set_input(gather_local(X, [(topB, 0, nrB, LAYERS[0][0])], net.buffer_shape(0)))
                if case["model"] == "gin":
                    net.forward()
                    out["out"] = net.buffer(len(LAYERS))
                    net.backward(gather_local(G, [(topA, 0, nrA, LAYERS[-1][2])], net.buffer_shape(len(LAYERS))))
                    out["dX"] = net.input_grad()
                    for l in range(len(LAYERS)):
                        for k in net.param_names():
                            out[f"g{l}_{k}"] = net.param_grad(l, k)
                else:  # train
                    lab = np.full(net.buffer_shape(len(LAYERS))[0], -1)
                    hi = min(topA + nrA, N)
                    lab[:hi - topA] = labels[topA:hi]
                    L = D.NodeLabels(net, lab, CLASSES)
                    opt = D.AdamW(lr=1e-2, max_grad_norm=0.5)
                    out["steps"] = np.array([tuple(net.train_step(L, opt)) for _ in range(3)], np.float64)
                    for l in range(len(LAYERS)):
                        for k in net.param_names():
                            out[f"p{l}_{k}"] = net.param(l, k)
        except (RuntimeError, ValueError) as e:
            out["error"] = f"{type(e).__name__}: {e}"
        np.savez(os.path.join(outdir, f"{name}_rank{rank}.npz"), **out)
        del S
    D.world_finalize()


if __name__ == "__main__":
    main()
