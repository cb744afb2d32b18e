"""Multi-process worker for the multi-rank training tests (launched through torch.distributed.run by
tests/test_training_multirank_gpu.py).  Per case every rank builds the model (a graph transformer, or GAT with the
case's attention kind), sets the global parameters and its rows of the input and of the labels, runs the case's train
steps and writes the per-step results and the trained parameters to <outdir>/<case>_rank<r>.npz, or the error every
rank must raise."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import gat_additive_oracle as gao  # noqa: E402
from tests import graph_transformer_block_oracle as gbo  # noqa: E402
from tests.mp_graph_transformer_worker import attr_of  # noqa: E402
from tests.mp_worker import gather_local  # noqa: E402


def global_inputs(case):
    """(params, X, labels) of a case, the same on every rank: params are GraphTransformer parameter dicts, or for GAT
    (weights, a1, a2)."""
    N, layers = 1 << case["logM"], [tuple(l) for l in case["layers"]]
    rng = np.random.default_rng(case["seed"] + 1)
    if case["model"] == "gt":
        params = gbo.random_params(layers, case["edge_dim"], case["beta"], case["ffn"], rng)
    else:
        params = ([[rng.uniform(-1, 1, (f, d)) / np.sqrt(f) for _ in range(H)] for f, d, H in layers],
                  *gao.attention_inputs(layers, case["seed"]))
    X = rng.uniform(0, 1, (N, layers[0][0]))
    C = layers[-1][1] * layers[-1][2]
    labels = rng.integers(0, C, N)
    labels[rng.random(N) < 0.2] = -1
    return params, X, labels


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
        N = 1 << logM
        per = N // world
        tr, tc, _ = orc.er_tuples(logM, npr, seed, per * rank, N if rank == world - 1 else per * (rank + 1))
        S = D.SpmatLocal.from_tuples(N, N, tr, tc, np.ones(len(tr)))
        alg = D.Algorithm(alg_name, S, layers[0][0], c)
        out = {}
        try:
            params, X, labels = global_inputs(case)
            if case["model"] == "gt":
                net = D.GraphTransformer(alg, layers, edge_dim=case["edge_dim"], beta=case["beta"], ffn_ratio=case["ffn"])
                for l, P in enumerate(params):
                    for pname, v in P.items():
                        net.set_param(l, pname, v)
            else:
                net = D.GAT(alg, layers, attention=case["kind"])
                # layouts that split R hold other weight shapes; there the train step must refuse before it reads them
                for l, (_, _, H) in enumerate(layers if not case.get("error") else []):
                    for h in range(H):
                        net.set_weight(l, h, params[0][l][h])
                        net.set_attention_vectors(l, h, params[1][l][h], params[2][l][h])
            topA, _, nrA, _ = alg.submatrices("A")[0]
            topB, _, nrB, _ = alg.submatrices("B")[0]
            if not case.get("error"):
                net.set_input(gather_local(X, [(topB, 0, nrB, layers[0][0])], net.buffer_shape(0)))
            if case["model"] == "gt" and case["edge_dim"]:
                net.set_edge_attributes(attr_of(*alg.entry_coordinates("A"), case["edge_dim"]),
                                        attr_of(*alg.entry_coordinates("B"), case["edge_dim"]))
            rows = net.buffer_shape(len(layers))[0]
            lab = -np.ones(rows, np.int64)
            hi = min(topA + rows, N)
            if not case.get("error"):
                lab[:hi - topA] = labels[topA:hi]
            nl = D.NodeLabels(net, lab, net.buffer_shape(len(layers))[1] if case.get("error") else layers[-1][1] * layers[-1][2])
            opt = D.AdamW(lr=1e-2, max_grad_norm=case.get("clip"))
            steps = []
            for t in range(case["steps"]):
                r = net.train_step(nl, opt, case["dropout"], 5 + t) if case["model"] == "gt" else net.train_step(nl, opt)
                steps.append(list(r))
            out["steps"] = np.array(steps)
            if case["model"] == "gt":
                for l in range(len(layers)):
                    for pname in net.param_names():
                        out[f"p{l}_{pname}"] = net.param(l, pname)
            else:
                for l, (_, _, H) in enumerate(layers):
                    for h in range(H):
                        out[f"w{l}_{h}"] = net.weight(l, h)
                        out[f"a1_{l}_{h}"], out[f"a2_{l}_{h}"] = net.attention_vectors(l, h)
        except RuntimeError as e:
            out["error"] = str(e)
        np.savez(os.path.join(outdir, f"{name}_rank{rank}.npz"), **out)
        del alg, S
    D.world_finalize()


if __name__ == "__main__":
    main()
