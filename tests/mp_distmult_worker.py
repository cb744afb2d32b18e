"""Multi-process worker for the multi-rank relational link-prediction tests (launched through torch.distributed.run by
tests/test_distmult_multirank_gpu.py).  Per case every rank builds the model's S from its row slice of an Erdos-Renyi
graph with hashed relations, and T_pos and T_neg from their round-robin shares of global triples, then runs the case:
the op (Algorithm.distmult_loss, a positive call and an accumulated negative call), relational link train steps of
R-GCN, or a refusal.  Results go to <outdir>/<case>_rank<r>.npz, or the error every rank must raise."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import rgcn_oracle as ro  # noqa: E402
from tests.mp_worker import gather_local  # noqa: E402

LAYERS = [(8, 8), (8, 8)]
R = 4


def global_inputs(case):
    """(S relations, positive triples, negative triples, H, rel, model params, X), the same on every rank."""
    N = 1 << case["logM"]
    rng = np.random.default_rng(case["seed"] + 3)
    trip = []
    for n in (4 * N, 3 * N):
        tr, tc, rels = rng.integers(0, N, n), rng.integers(0, N, n), rng.integers(0, R, n).astype(np.float64)
        tr[:9], tc[:9] = tr[9:18], tc[9:18]  # the same pairs under other relations
        rels[:9] = (rels[9:18] + 1) % R
        tr[20:60] = 3  # a hub row
        trip.append((tr.astype(np.int64), tc.astype(np.int64), rels))
    H = rng.standard_normal((N, case["r"])) / 2
    H[5] *= 10.0
    rel = rng.standard_normal((R, case["r"]))
    params = ro.random_params(LAYERS, R, rng)
    X = rng.uniform(-1, 1, (N, LAYERS[0][0]))
    return trip[0], trip[1], H, rel, params, X


def s_relations(rows, cols, N):
    return ((rows * 7 + cols * 3) % R).astype(np.float64)


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
        sr, sc_ = np.asarray(sr, np.int64), np.asarray(sc_, np.int64)
        S = D.SpmatLocal.from_tuples(N, N, sr, sc_, s_relations(sr, sc_, N))
        f0 = LAYERS[0][0]
        alg = D.Algorithm(alg_name, S, f0, c)
        pos, neg, H, rel, params, X = global_inputs(case)
        if case.get("bad_rank") == rank:
            rels = neg[2].copy()
            rels[rank::world][0] = float(R)
            neg = (neg[0], neg[1], rels)
        out = {}
        try:
            mk = lambda t: D.Algorithm(alg_name, D.SpmatLocal.from_tuples(N, N, *(a[rank::world] for a in t)), f0, c)  # noqa: E731
            alg_pos, alg_neg = mk(pos), mk(neg)
            topA, _, nrA, _ = alg.submatrices("A")[0]
            if case["model"] == "op":
                r = case["r"]
                Hl = D.Dense.create(alg_pos.like_A_matrix().shape[0], r)
                Hl.from_host(gather_local(H, [(topA, 0, nrA, r)], Hl.shape))
                Dd = D.Dense.create(R, r)
                Dd.from_host(rel)
                dH, dD = D.Dense.create(*Hl.shape), D.Dense.create(R, r)
                sp, sn = alg_pos.like_S_values(), alg_neg.like_S_values()
                inv = 1.0 / (len(pos[0]) + len(neg[0]))
                res = []
                for _ in range(2):  # the second pass repeats the first
                    res.append(alg_pos.distmult_loss(Hl, Hl, Dd, R, 1.0, inv, dH, dH, dD, sp))
                    res.append(alg_neg.distmult_loss(Hl, Hl, Dd, R, 0.0, inv, dH, dH, dD, sn, accumulate=True))
                out["res"] = np.array(res, np.float64)
                out["dH"], out["dD"], out["top"] = dH.to_host(), dD.to_host(), np.array([topA])
                out["sp"], out["sn"] = sp.to_host(), sn.to_host()
                out["erp"], out["ecp"] = alg_pos.entry_coordinates("A")
                out["ern"], out["ecn"] = alg_neg.entry_coordinates("A")
            else:
                net = D.RGCN(alg, LAYERS, num_relations=R, num_bases=case.get("bases"))
                if case.get("bases"):
                    from tests import rgcn_basis_oracle as bo
                    params = bo.random_params(LAYERS, R, case["bases"], np.random.default_rng(seed + 9))
                for l, P in enumerate(params):
                    for k, v in P.items():
                        net.set_param(l, k, v)
                topB, _, nrB, _ = alg.submatrices("B")[0]
                net.set_input(gather_local(X, [(topB, 0, nrB, f0)], net.buffer_shape(0)))
                dec = D.DistMultDecoder(net, R)
                dec.set_param("rel", rel[:, :LAYERS[-1][1]])
                t = D.RelationalLinkTargets(net, alg_pos, alg_neg, R)
                opt = D.AdamW(lr=1e-2, max_grad_norm=1.0)
                out["steps"] = np.array([list(net.relational_link_train_step(dec, t, opt)) for _ in range(case["steps"])])
                out["rel"], out["drel"] = dec.param("rel"), dec.param_grad("rel")
                for l in range(len(LAYERS)):
                    for pname in net.param_names():
                        out[f"p{l}_{pname}"] = net.param(l, pname)
        except RuntimeError as e:
            out["error"] = str(e)
        np.savez(os.path.join(outdir, f"{name}_rank{rank}.npz"), **out)
        del alg, S
    D.world_finalize()


if __name__ == "__main__":
    main()
