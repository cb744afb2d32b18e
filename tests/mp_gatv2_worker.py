"""Multi-process worker for the multi-rank GATv2 tests (launched through torch.distributed.run by
tests/test_gatv2_multirank_gpu.py).  Every rank builds the requested algorithm through the driver ABI, then runs a
GATv2 GAT forward + backward on its rows of the global inputs and writes the results -- or, on a layout without GATv2
attention, the errors that gatv2_scores, gatv2_backward and the forward pass raised -- to <outdir>/<case>_rank<r>.npz.

Transports as in tests/mp_worker.py: "gloo" (ranks sharing one GPU), "nccl" (one GPU per rank)."""
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests.gatv2_oracle import attention_inputs  # noqa: E402
from tests.mp_gat_backward_worker import output_grad  # noqa: E402
from tests.mp_worker import gat_inputs, gather_local, sval  # noqa: E402


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
        a = attention_inputs(layers, seed)
        alg = D.Algorithm(alg_name, S, layers[0][0], c)
        net = D.GAT(alg, layers, case["alpha"], attention="gatv2")
        out = {}
        if case.get("rejected"):
            # a layout without GATv2 attention: every entry point must refuse before any launch
            A, B, av = alg.like_A_matrix(), alg.like_B_matrix(), vec(layers[0][0])
            for key, call in (("scores_error", lambda: alg.gatv2_scores(A, B, av, alg.like_S_values(0.0), "A")),
                              ("backward_error", lambda: alg.gatv2_backward(A, B, av, alg.like_S_values(0.0), alg.like_ST_values(0.0),
                                                                            A, B, vec(1))),
                              ("gat_error", net.forward)):
                try:
                    call()
                except RuntimeError as e:
                    out[key] = str(e)
            np.savez(os.path.join(outdir, f"{name}_rank{rank}.npz"), **out)
            del net, alg, S
            continue
        # this rank's rows of the global input, the global weights, attention vectors and output gradient
        topB, _, nrB, _ = alg.submatrices("B")[0]
        topA, _, nrA, _ = alg.submatrices("A")[0]
        out.update(topA=topA, nrA=nrA, topB=topB, nrB=nrB)
        for i, (_, fph, heads) in enumerate(layers):
            for h in range(heads):
                net.set_weight(i, h, weights[i][h])
                net.set_attention_vectors(i, h, a[i][h], np.zeros(fph))
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
                    out[f"da_{i}_{h}"] = net.attention_grads(i, h)[0]
        except RuntimeError as e:
            out["gat_error"] = str(e)
        np.savez(os.path.join(outdir, f"{name}_rank{rank}.npz"), **out)
        del net, alg, S
    D.world_finalize()


if __name__ == "__main__":
    main()
