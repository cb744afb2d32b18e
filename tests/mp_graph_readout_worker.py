"""Multi-process worker for the multi-rank graph readout tests (launched through torch.distributed.run by
tests/test_graph_readout_multirank_gpu.py).  Per case every rank builds S from its row slice of an Erdos-Renyi graph,
a model on it, and a GraphReadout from its slice of one global batch vector, then runs the case: the op
(GraphReadout.pool / pool_backward on a given H), graph train steps of GraphSAGE or the graph transformer, or a
refusal.  Results go to <outdir>/<case>_rank<r>.npz, or the error every rank must raise."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import graph_sage_oracle as gso  # noqa: E402
from tests import graph_transformer_oracle as gto  # noqa: E402
from tests.mp_worker import gather_local  # noqa: E402

F0 = 8  # the input width: R divisible by p / c on every layout
SAGE_LAYERS = [(F0, 8), (8, 4)]
GT_LAYERS = [(F0, 4, 2), (8, 2, 2)]
CLASSES = 3


def global_inputs(case):
    """(batch over the N rows, G, labels, H for the op, model params, head (W, b), X), the same on every rank.  Graphs
    are runs of 3..40 rows with shuffled ids, so they straddle rank boundaries; rows N/2 - 4 .. N/2 + 3 belong to one
    graph, and H rows N/2 - 2 and N/2 + 1 (on two ranks) are equal and its maximum: a max tie across ranks.  The last
    graph is empty; empty_rank leaves that rank's rows in no graph."""
    N, p = 1 << case["logM"], case["p"]
    rng = np.random.default_rng(case["seed"] + 5)
    batch = np.empty(N, np.int64)
    g = i = 0
    while i < N:
        L = int(rng.integers(3, 41))
        batch[i:i + L] = g
        g, i = g + 1, i + L
    batch = rng.permutation(g)[batch]
    batch[rng.random(N) < 0.1] = -1
    h = N // 2
    batch[h - 4:h + 4] = batch[h - 5] if batch[h - 5] >= 0 else 0
    if case.get("empty_rank") is not None:
        per = N // p
        batch[per * case["empty_rank"]:per * (case["empty_rank"] + 1)] = -1
    G = g + 1
    labels = rng.integers(0, CLASSES, G)
    labels[rng.random(G) < 0.2] = -1
    r = case.get("r", 16)
    H = rng.standard_normal((N, r))
    H[h - 2] = H[h + 1] = 5.0 + rng.random(r)
    if case["model"] == "gt":
        params = gto.random_params(GT_LAYERS, 0, False, rng)
        width = GT_LAYERS[-1][1] * GT_LAYERS[-1][2]
    else:
        params = gso.random_params(SAGE_LAYERS, rng)
        width = SAGE_LAYERS[-1][1]
    head = (rng.uniform(-1, 1, (width, CLASSES)), rng.uniform(-0.5, 0.5, CLASSES)) if case.get("head") else None
    X = rng.uniform(-1, 1, (N, F0))
    return batch, G, labels, H, params, head, X


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
        sr, sc_, _ = orc.er_tuples(logM, 5, seed, per * rank, N if rank == world - 1 else per * (rank + 1))
        S = D.SpmatLocal.from_tuples(N, N, sr, sc_, np.ones(len(sr)))
        alg = D.Algorithm(alg_name, S, F0, c)
        batch, G, labels, H, params, head, X = global_inputs(case)
        out = {}
        try:
            if case["model"] == "gat":  # a model every layout builds, for the readout's layout refusal
                net = D.GAT(alg, [(F0, 4, 1)])
            elif case["model"] == "op":
                net = D.GraphSAGE(alg, [(F0, case["r"])], aggr="sum")
            elif case["model"] == "gt":
                net = D.GraphTransformer(alg, GT_LAYERS)
                for l, P in enumerate(params):
                    for k, v in P.items():
                        net.set_param(l, k, v)
            else:
                net = D.GraphSAGE(alg, SAGE_LAYERS, aggr=case["aggr"])
                for l, P in enumerate(params):
                    for k, v in P.items():
                        net.set_param(l, k, v)
            topA, _, nrA, _ = alg.submatrices("A")[0]
            rows_out = net.buffer_shape(len(net.layers))[0]
            local = np.full(rows_out, -1, np.int64)
            hi = min(topA + rows_out, N)
            local[:hi - topA] = batch[topA:hi]
            if case.get("bad_batch_rank") == rank:
                local[0] = G
            Gl = G + 1 if case.get("bad_g_rank") == rank else G
            ro = D.GraphReadout(net, local, Gl, pool=case["pool"], num_classes=CLASSES if head else None)
            out["top"] = np.array([topA, rows_out])
            if case["model"] == "op":
                r = case["r"]
                Hd = D.Dense.create(rows_out, r)
                Hd.from_host(gather_local(H, [(topA, 0, rows_out, r)], (rows_out, r)))
                P = ro.pool(Hd)
                dPh = np.random.default_rng(seed + 9).standard_normal((G, r))
                dP = D.Dense.create(G, r)
                dP.from_host(dPh)
                out["P"], out["dH"] = P.to_host(), ro.pool_backward(dP).to_host()
                out["again"] = ro.pool(Hd).to_host()
            else:
                if head:
                    ro.set_param("weight", head[0])
                    ro.set_param("bias", head[1])
                topB, _, nrB, _ = alg.submatrices("B")[0]
                net.set_input(gather_local(X, [(topB, 0, nrB, F0)], net.buffer_shape(0)))
                lab = labels.copy()
                if case.get("bad_labels_rank") == rank:
                    lab[0] = (lab[0] + 1) % CLASSES
                gl = D.GraphLabels(ro, lab, ro.num_classes)
                opt = D.AdamW(lr=1e-2, max_grad_norm=0.5)
                steps = []
                for s in range(case["steps"]):
                    res = net.graph_train_step(ro, gl, opt, case["dropout"], 5 + s) if case["model"] == "gt" else \
                        net.graph_train_step(ro, gl, opt)
                    steps.append(list(res))
                out["steps"] = np.array(steps)
                for l in range(len(net.layers)):
                    for pname in net.param_names():
                        out[f"p{l}_{pname}"] = net.param(l, pname)
                for pname in ro.param_names():
                    out[f"head_{pname}"] = ro.param(pname)
                    out[f"headgrad_{pname}"] = ro.param_grad(pname)
                out["logits"] = net.graph_evaluate(ro, gl)[3]
        except RuntimeError as e:
            out["error"] = str(e)
        np.savez(os.path.join(outdir, f"{name}_rank{rank}.npz"), **out)
        del alg, S
    D.world_finalize()


if __name__ == "__main__":
    main()
