"""Multi-process worker for the multi-rank attention-bias tests (launched through torch.distributed.run by
tests/test_sparse_attention_bias_multirank_gpu.py).  Every rank builds the requested algorithm through the driver ABI,
builds its A- and B-order biases from Algorithm.entry_coordinates with bias_of (per head or shared), runs
Algorithm.sparse_attention and sparse_attention_backward with the case's dropout and seed on its rows of the global Q,
K, V and dZ (tests/mp_sparse_attention_worker.global_inputs), and writes its rows of Z, L, dQ, dK and dV, its entry
coordinates and both dbias vectors to <outdir>/<case>_rank<r>.npz -- or the error every rank must raise.

Transports as in tests/mp_worker.py: "gloo" (ranks sharing one GPU), "nccl" (one GPU per rank)."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests.mp_sparse_attention_worker import global_inputs  # noqa: E402
from tests.mp_worker import gather_local, sval  # noqa: E402


def bias_of(rows, cols, h):
    """b(u, v) for head h: a function of the global S-row and S-column only, -inf on about 1 in 9 pairs and every pair
    of rows 5, 16, 27, ... (rows masked throughout), +-600 on alternate rows."""
    rows, cols = np.asarray(rows), np.asarray(cols)
    b = np.sin(0.37 * rows + 1.3 * cols + 0.5 * h) * 2.0 + np.where(rows % 2 == 0, 600.0, -600.0)
    b[((rows * 7 + cols * 3 + h) % 9 == 4) | (rows % 11 == 5)] = -np.inf
    return b


def biases(rows, cols, heads, shared):
    return np.concatenate([bias_of(rows, cols, h) for h in ([0] if shared else range(heads))])


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
        name, alg_name, c, logM, npr, seed, heads, d, p, mask_seed, shared = (
            case[k] for k in ("name", "alg", "c", "logM", "npr", "seed", "heads", "d", "dropout", "mask_seed", "shared"))
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
            vecs = []
            for rr, cc in ((rA, cA), (rB, cB)):
                b = biases(rr, cc, heads, shared)
                v = D.Vec.create(len(b))
                v.from_host(b)
                vecs.append(v)
            dbA, dbB = D.Vec.create(0), D.Vec.create(0)
            alg.sparse_attention(Q, K, V, Z, L, heads, dropout=p, seed=mask_seed, bias=vecs[0])
            alg.sparse_attention_backward(Q, K, V, Z, L, dZ, dQ, dK, dV, heads, dropout=p, seed=mask_seed, bias=vecs[0],
                                          bias_B=vecs[1], dbias=dbA, dbias_B=dbB)
            for key, m in (("Z", Z), ("L", L), ("dQ", dQ), ("dK", dK), ("dV", dV), ("dbA", dbA), ("dbB", dbB)):
                out[key] = m.to_host()
            out.update(rA=rA, cA=cA, rB=rB, cB=cB)
        except RuntimeError as e:
            out["error"] = str(e)
        np.savez(os.path.join(outdir, f"{name}_rank{rank}.npz"), **out)
        del alg, S
    D.world_finalize()


if __name__ == "__main__":
    main()
