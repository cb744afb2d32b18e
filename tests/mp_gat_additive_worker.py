"""Multi-process worker for the multi-rank additive-attention tests (launched through torch.distributed.run by
tests/test_gat_additive_multirank_gpu.py).  Every rank builds the requested algorithm through the driver ABI, then
  * finds the (row, col) of every entry of its A-order and B-order value vectors from SDDMMs of index columns, and
    the same through additive_scores of index node vectors (the row and column keys),
  * takes the world row and column sums of an A-order vector that is a function of (row, col),
  * runs an additive-attention GAT forward + backward on its rows of the global inputs,
and writes the results -- or the errors raised -- to <outdir>/<case>_rank<r>.npz.

Transports as in tests/mp_worker.py: "gloo" (ranks sharing one GPU), "nccl" (one GPU per rank)."""
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests.gat_additive_oracle import attention_inputs  # noqa: E402
from tests.mp_edge_softmax_worker import coords  # noqa: E402
from tests.mp_gat_backward_worker import output_grad  # noqa: E402
from tests.mp_worker import gat_inputs, gather_local, sval  # noqa: E402


def summand(r, c):
    """The A-order vector whose row and column sums a case takes."""
    return np.cos(0.3 * np.asarray(r, np.float64) + 0.7 * np.asarray(c, np.float64))


def main():
    cases = json.loads(sys.argv[1])
    outdir = sys.argv[2]
    transport = sys.argv[3]
    import torch
    ngpu = torch.cuda.device_count()
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")) % ngpu if transport == "nccl" else 0)
    from distributed_sddmm_b200 import driver as D
    from distributed_sddmm_b200 import lib
    from oracle import hnh_oracle as orc
    rank, world = D.world_init(transport)

    def vec(n, value=0.0):
        h = C.c_void_p()
        D.check(lib().hnhd_vec_create(n, value, C.byref(h)))
        return D.Vec(h)

    for case in cases:
        name, alg_name, c, logM, npr, seed = (case[k] for k in ("name", "alg", "c", "logM", "npr", "seed"))
        N = 1 << logM
        per = N // world
        tr, tc, _ = orc.er_tuples(logM, npr, seed, per * rank, N if rank == world - 1 else per * (rank + 1))
        S = D.SpmatLocal.from_tuples(N, N, tr, tc, sval(tr, tc))
        layers, X0, weights = gat_inputs(N, case["layers"], seed)
        a1, a2 = attention_inputs(layers, seed)
        alg = D.Algorithm(alg_name, S, layers[0][0], c)
        out = {}
        if case.get("rejected"):
            # a layout without additive attention: every entry point must refuse before any launch
            net = D.GAT(alg, layers, case["alpha"], attention="additive")
            zero = vec(N)
            for key, call in (("scores_error", lambda: alg.additive_scores(zero, zero, alg.like_S_values(0.0), "A")),
                              ("sums_error", lambda: alg.edge_sums(alg.like_S_values(0.0), vec(N), vec(N))),
                              ("gat_error", net.forward)):
                try:
                    call()
                except RuntimeError as e:
                    out[key] = str(e)
            np.savez(os.path.join(outdir, f"{name}_rank{rank}.npz"), **out)
            del net, alg, S
            continue
        # row and column keys in both orders, and the world row / column sums of an A-order vector
        try:
            zero, index = vec(N), vec(N)
            index.from_host(np.arange(N, dtype=np.float64))
            for mode in ("A", "B"):
                r, cc = coords(alg, mode)
                v = (alg.like_S_values if mode == "A" else alg.like_ST_values)(-1.0)
                alg.additive_scores(index, zero, v, mode)
                kr = v.to_host()
                alg.additive_scores(zero, index, v, mode)
                out.update({f"{mode}_rows": r, f"{mode}_cols": cc, f"{mode}_row_keys": kr, f"{mode}_col_keys": v.to_host()})
            v = alg.like_S_values(0.0)
            v.from_host(summand(out["A_rows"], out["A_cols"]))
            rs, cs = vec(N), vec(N)
            alg.edge_sums(v, rs, cs)
            out.update(row_sums=rs.to_host(), col_sums=cs.to_host())
        except RuntimeError as e:
            out["keys_error"] = str(e)
        # additive GAT (made after the SDDMMs above: it changes the algorithm's R): this rank's rows of the global
        # input, the global weights, attention vectors and output gradient
        net = D.GAT(alg, layers, case["alpha"], attention="additive")
        topB, _, nrB, _ = alg.submatrices("B")[0]
        topA, _, nrA, _ = alg.submatrices("A")[0]
        out.update(topA=topA, nrA=nrA, topB=topB, nrB=nrB)
        for i, (_, _, heads) in enumerate(layers):
            for h in range(heads):
                net.set_weight(i, h, weights[i][h])
                net.set_attention_vectors(i, h, a1[i][h], a2[i][h])
        net.set_input(gather_local(X0, [(topB, 0, nrB, layers[0][0])], net.buffer_shape(0)))
        out_width = layers[-1][1] * layers[-1][2]
        G = gather_local(output_grad(N, out_width, seed), [(topA, 0, nrA, out_width)], net.buffer_shape(len(layers)))
        try:
            net.forward()
            out["out"] = net.buffer(len(layers))
            net.backward(G)
            out["dX0"] = net.input_grad()
            for i, (_, _, heads) in enumerate(layers):
                for h in range(heads):
                    out[f"dW_{i}_{h}"] = net.weight_grad(i, h)
                    out[f"da1_{i}_{h}"], out[f"da2_{i}_{h}"] = net.attention_grads(i, h)
        except RuntimeError as e:
            out["gat_error"] = str(e)
        np.savez(os.path.join(outdir, f"{name}_rank{rank}.npz"), **out)
        del net, alg, S
    D.world_finalize()


if __name__ == "__main__":
    main()
