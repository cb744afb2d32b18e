"""Multi-process worker for the multi-rank graph transformer block tests (launched through torch.distributed.run by
tests/test_graph_transformer_block_multirank_gpu.py).  As tests/mp_graph_transformer_worker.py, with the case's
ffn_ratio and the block parameters of tests/graph_transformer_block_oracle.random_params: every rank writes its rows
of the output and the input gradient and every parameter gradient to <outdir>/<case>_rank<r>.npz, or the error every
rank must raise."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import graph_transformer_block_oracle as gbo  # noqa: E402
from tests.mp_graph_transformer_worker import attr_of  # noqa: E402
from tests.mp_worker import gather_local  # noqa: E402


def global_inputs(N, layers, edge_dim, beta, ffn, seed):
    """(params, X, G) of a case: the same on every rank."""
    rng = np.random.default_rng(seed)
    params = gbo.random_params(layers, edge_dim, beta, ffn, rng)
    X = rng.uniform(-1, 1, (N, layers[0][0]))
    G = rng.uniform(-1, 1, (N, layers[-1][1] * layers[-1][2]))
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
        name, alg_name, c, logM, npr, seed = (case[k] for k in ("name", "alg", "c", "logM", "npr", "seed"))
        layers = [tuple(l) for l in case["layers"]]
        edge_dim, beta, ffn, p, mask_seed = case["edge_dim"], case["beta"], case["ffn"], case["dropout"], case["mask_seed"]
        N = 1 << logM
        per = N // world
        tr, tc, _ = orc.er_tuples(logM, npr, seed, per * rank, N if rank == world - 1 else per * (rank + 1))
        S = D.SpmatLocal.from_tuples(N, N, tr, tc, np.ones(len(tr)))
        alg = D.Algorithm(alg_name, S, layers[0][0], c)
        out = {}
        try:
            net = D.GraphTransformer(alg, layers, edge_dim=edge_dim, beta=beta, ffn_ratio=ffn)
            params, X, G = global_inputs(N, layers, edge_dim, beta, ffn, seed + 1)
            for l, P in enumerate(params):
                for pname, v in P.items():
                    net.set_param(l, pname, v)
            topA, _, nrA, _ = alg.submatrices("A")[0]
            topB, _, nrB, _ = alg.submatrices("B")[0]
            out.update(topA=topA, nrA=nrA, topB=topB, nrB=nrB)
            f, r = layers[0][0], layers[-1][1] * layers[-1][2]
            net.set_input(gather_local(X, [(topB, 0, nrB, f)], net.buffer_shape(0)))
            if edge_dim:
                net.set_edge_attributes(attr_of(*alg.entry_coordinates("A"), edge_dim),
                                        attr_of(*alg.entry_coordinates("B"), edge_dim))
            net.forward(p, mask_seed)
            net.backward(gather_local(G, [(topA, 0, nrA, r)], net.buffer_shape(len(layers))))
            out["Y"] = net.buffer(len(layers))
            out["dX"] = net.input_grad()
            for l in range(len(layers)):
                for pname in net.param_names():
                    out[f"g{l}_{pname}"] = net.param_grad(l, pname)
        except RuntimeError as e:
            out["error"] = str(e)
        np.savez(os.path.join(outdir, f"{name}_rank{rank}.npz"), **out)
        del alg, S
    D.world_finalize()


if __name__ == "__main__":
    main()
