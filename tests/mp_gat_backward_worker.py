"""Multi-process worker for the multi-rank GAT backward tests (launched through torch.distributed.run by
tests/test_gat_backward_multirank_gpu.py).  Every rank builds the requested algorithm and GAT through the driver ABI,
runs forward + backward on its own rows of the global inputs and writes its input gradient rows, every weight
gradient -- or the error the backward pass raised -- to <outdir>/<case>_rank<r>.npz.

Transports as in tests/mp_worker.py: "gloo" (ranks sharing one GPU), "nccl" (one GPU per rank)."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests.mp_worker import gat_inputs, gather_local, sval  # noqa: E402


def output_grad(N, width, seed):
    """The global dL/d(network output) of a case."""
    return np.random.default_rng(seed + 55).uniform(-1, 1, (N, width))


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
        N = 1 << logM
        per = N // world  # tuples dealt in contiguous row slices, coordinate-dependent values (ignored by GAT)
        tr, tc, _ = orc.er_tuples(logM, npr, seed, per * rank, N if rank == world - 1 else per * (rank + 1))
        S = D.SpmatLocal.from_tuples(N, N, tr, tc, sval(tr, tc))
        layers, X0, weights = gat_inputs(N, case["layers"], seed)
        alg = D.Algorithm(alg_name, S, layers[0][0], c)
        net = D.GAT(alg, layers, case["alpha"])
        topB, _, nrB, _ = alg.submatrices("B")[0]
        topA, _, nrA, _ = alg.submatrices("A")[0]
        out = dict(topB=topB, nrB=nrB)
        if case.get("forward", True):
            # full-width rows: this rank's rows of the global input, the global weights, the global output gradient
            for i, (_, _, heads) in enumerate(layers):
                for h in range(heads):
                    net.set_weight(i, h, weights[i][h])
            net.set_input(gather_local(X0, [(topB, 0, nrB, layers[0][0])], net.buffer_shape(0)))
            out_width = layers[-1][1] * layers[-1][2]
            G = gather_local(output_grad(N, out_width, seed), [(topA, 0, nrA, out_width)], net.buffer_shape(len(layers)))
            net.forward()
        else:
            G = np.zeros(net.buffer_shape(len(layers)))
        try:
            net.backward(G)
            out["dX0"] = net.input_grad()
            for i, (_, _, heads) in enumerate(layers):
                for h in range(heads):
                    out[f"dW_{i}_{h}"] = net.weight_grad(i, h)
        except RuntimeError as e:
            out["error"] = str(e)
        np.savez(os.path.join(outdir, f"{name}_rank{rank}.npz"), **out)
        del net, alg, S
    D.world_finalize()


if __name__ == "__main__":
    main()
