"""Multi-process worker for the multi-rank link-prediction tests (launched through torch.distributed.run by
tests/test_link_prediction_multirank_gpu.py).  Per case every rank builds the model's S from its row slice of an
Erdos-Renyi graph and the target matrix T from its round-robin share of global targets, then runs the case: the op
(Algorithm.link_loss with H_A = H_B and dH_A = dH_B), link train steps of a model, or a refusal.  Results go to
<outdir>/<case>_rank<r>.npz, or the error every rank must raise."""
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

GT_LAYERS = [(6, 4, 2), (8, 8, 1)]
GAT_LAYERS = [(8, 4, 2), (8, 6, 1)]


def global_inputs(case):
    """(T rows, T cols, targets, H, model params, X), the same on every rank."""
    N = 1 << case["logM"]
    rng = np.random.default_rng(case["seed"] + 3)
    n = 6 * N
    tr, tc = rng.integers(0, N, n), rng.integers(0, N, n)
    tr[:9], tc[:9] = tr[9:18], tc[9:18]  # duplicates
    tr[20:60] = 3  # a hub row
    y = rng.choice([0.0, 1.0, 0.25], n)
    y[:9] = y[9:18]
    H = rng.standard_normal((N, case["r"])) / 2
    H[5] *= 30.0
    if case["model"] == "gat":
        params = ([[rng.uniform(-1, 1, (f, d)) / np.sqrt(f) for _ in range(Hh)] for f, d, Hh in GAT_LAYERS],
                  *gao.attention_inputs(GAT_LAYERS, case["seed"]))
        X = rng.uniform(0, 1, (N, GAT_LAYERS[0][0]))
    else:
        params = gbo.random_params(GT_LAYERS, 2, True, 1, rng)
        X = rng.uniform(-1, 1, (N, GT_LAYERS[0][0]))
    return tr.astype(np.int64), tc.astype(np.int64), y, H, params, X


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
        f0 = GAT_LAYERS[0][0] if case["model"] in ("gat", "op") else GT_LAYERS[0][0]  # 8: R divisible by p / c everywhere
        alg = D.Algorithm(alg_name, S, f0, c)
        tr, tc, y, H, params, X = global_inputs(case)
        if case.get("bad_rank") == rank:
            y = y.copy()
            y[rank::world][0] = 1.5
        out = {}
        try:
            T = D.SpmatLocal.from_tuples(N, N, tr[rank::world], tc[rank::world], y[rank::world])
            algT = D.Algorithm(case.get("t_alg", alg_name), T, f0, case.get("t_c", c))
            topA, _, nrA, _ = alg.submatrices("A")[0]
            if case["model"] == "op":
                Hl = D.Dense.create(algT.like_A_matrix().shape[0], case["r"])
                Hl.from_host(gather_local(H, [(topA, 0, nrA, case["r"])], Hl.shape))
                dH = D.Dense.create(*Hl.shape)
                scores = algT.like_S_values()
                res = algT.link_loss(Hl, Hl, dH, dH, scores)
                again = algT.link_loss(Hl, Hl, dH, dH, scores)
                out["res"], out["again"] = np.array(res, np.float64), np.array(again, np.float64)
                out["dH"], out["scores"], out["top"] = dH.to_host(), scores.to_host(), np.array([topA])
                out["er"], out["ec"] = algT.entry_coordinates("A")
            else:
                if case["model"] == "gt":
                    net = D.GraphTransformer(alg, GT_LAYERS, edge_dim=2, beta=True, ffn_ratio=1)
                    for l, P in enumerate(params):
                        for k, v in P.items():
                            net.set_param(l, k, v)
                else:
                    net = D.GAT(alg, GAT_LAYERS, attention=case["kind"])
                    for l, (_, _, Hh) in enumerate(GAT_LAYERS if not case.get("error") else []):
                        for h in range(Hh):
                            net.set_weight(l, h, params[0][l][h])
                            net.set_attention_vectors(l, h, params[1][l][h], params[2][l][h])
                topB, _, nrB, _ = alg.submatrices("B")[0]
                if not case.get("error"):
                    net.set_input(gather_local(X, [(topB, 0, nrB, f0)], net.buffer_shape(0)))
                    if case["model"] == "gt":
                        net.set_edge_attributes(attr_of(*alg.entry_coordinates("A"), 2), attr_of(*alg.entry_coordinates("B"), 2))
                t = D.LinkTargets(net, algT)
                opt = D.AdamW(lr=1e-2, max_grad_norm=case.get("clip"))
                steps = []
                for s in range(case["steps"]):
                    r = net.link_train_step(t, opt, case["dropout"], 5 + s) if case["model"] == "gt" else net.link_train_step(t, opt)
                    steps.append(list(r))
                out["steps"] = np.array(steps)
                if case["model"] == "gt":
                    for l in range(len(GT_LAYERS)):
                        for pname in net.param_names():
                            out[f"p{l}_{pname}"] = net.param(l, pname)
                else:
                    for l, (_, _, Hh) in enumerate(GAT_LAYERS):
                        for h in range(Hh):
                            out[f"w{l}_{h}"] = net.weight(l, h)
                            out[f"a1_{l}_{h}"], out[f"a2_{l}_{h}"] = net.attention_vectors(l, h)
        except RuntimeError as e:
            out["error"] = str(e)
        np.savez(os.path.join(outdir, f"{name}_rank{rank}.npz"), **out)
        del alg, S
    D.world_finalize()


if __name__ == "__main__":
    main()
