"""Multi-process worker for the multi-rank edge-feature attention tests (launched through torch.distributed.run by
tests/test_sparse_attention_edge_multirank_gpu.py).  Every rank builds the requested algorithm through the driver ABI,
builds its A- and B-order edge features from Algorithm.entry_coordinates with edge_of (and, when the case asks, a
shared bias with bias_of), runs Algorithm.sparse_attention and sparse_attention_backward with the case's dropout and
seed on its rows of the global Q, K, V and dZ (tests/mp_sparse_attention_worker.global_inputs), and writes its rows of
Z, L, dQ, dK and dV, its entry coordinates and its dE to <outdir>/<case>_rank<r>.npz -- or the error every rank must
raise.

Transports as in tests/mp_worker.py: "gloo" (ranks sharing one GPU), "nccl" (one GPU per rank)."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests.mp_sparse_attention_bias_worker import bias_of  # noqa: E402
from tests.mp_sparse_attention_worker import global_inputs  # noqa: E402
from tests.mp_worker import gather_local, sval  # noqa: E402


def edge_of(rows, cols, r):
    """e(u, v): r columns that are a function of the global S-row and S-column only."""
    rows, cols = np.asarray(rows, np.float64), np.asarray(cols, np.float64)
    return np.cos(0.31 * rows[:, None] + 0.73 * cols[:, None] + 0.45 * np.arange(r)[None, :])


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
        name, alg_name, c, logM, npr, seed, heads, d, p, mask_seed, with_bias = (
            case[k] for k in ("name", "alg", "c", "logM", "npr", "seed", "heads", "d", "dropout", "mask_seed", "bias"))
        N = 1 << logM
        r = heads * d
        per = N // world
        tr, tc, _ = orc.er_tuples(logM, npr, seed, per * rank, N if rank == world - 1 else per * (rank + 1))
        S = D.SpmatLocal.from_tuples(N, N, tr, tc, sval(tr, tc))
        alg = D.Algorithm(alg_name, S, r, c)
        dims = alg.dims
        Q, K, V, dZ = alg.like_A_matrix(), alg.like_B_matrix(), alg.like_B_matrix(), alg.like_A_matrix()
        Z, dQ, dK, dV = alg.like_A_matrix(), alg.like_A_matrix(), alg.like_B_matrix(), alg.like_B_matrix()
        L = D.Dense.create(dims.localArows, heads)
        Qg, Kg, Vg, dZg = global_inputs(N, r, seed)
        topA, _, nrA, _ = alg.submatrices("A")[0]
        topB, _, nrB, _ = alg.submatrices("B")[0]
        out = dict(topA=topA, nrA=nrA, topB=topB, nrB=nrB)
        for m, g, top, nr in ((Q, Qg, topA, nrA), (dZ, dZg, topA, nrA), (K, Kg, topB, nrB), (V, Vg, topB, nrB)):
            m.from_host(gather_local(g, [(top, 0, nr, r)], m.shape))
        try:
            rA, cA = alg.entry_coordinates("A")
            rB, cB = alg.entry_coordinates("B")
            edges = []
            for rr, cc in ((rA, cA), (rB, cB)):
                e = edge_of(rr, cc, r)
                m = D.Dense.create(*e.shape)
                m.from_host(e)
                edges.append(m)
            bias = [None, None]
            if with_bias:
                for i, (rr, cc) in enumerate(((rA, cA), (rB, cB))):
                    bias[i] = D.Vec.create(len(rr))
                    bias[i].from_host(bias_of(rr, cc, 0))
            dE = D.Dense.create(1, 1)
            alg.sparse_attention(Q, K, V, Z, L, heads, dropout=p, seed=mask_seed, bias=bias[0], edge=edges[0])
            alg.sparse_attention_backward(Q, K, V, Z, L, dZ, dQ, dK, dV, heads, dropout=p, seed=mask_seed, bias=bias[0],
                                          bias_B=bias[1], edge=edges[0], edge_B=edges[1], dedge=dE)
            for key, m in (("Z", Z), ("L", L), ("dQ", dQ), ("dK", dK), ("dV", dV), ("dE", dE)):
                out[key] = m.to_host()
            out.update(rA=rA, cA=cA, rB=rB, cB=cB)
        except RuntimeError as e:
            out["error"] = str(e)
        np.savez(os.path.join(outdir, f"{name}_rank{rank}.npz"), **out)
        del alg, S
    D.world_finalize()


if __name__ == "__main__":
    main()
