"""Multi-process worker for the multi-rank edge-softmax tests (launched through torch.distributed.run by
tests/test_edge_softmax_multirank_gpu.py).  Every rank builds the requested algorithm through the driver ABI, then
  * finds the (row, col) of every entry of its A-order and B-order value vectors from SDDMMs of index columns,
  * runs edge_softmax and edge_softmax_backward on scores that are a function of (row, col), with -inf on the
    entries of `masked` when the case asks for a mask,
  * runs a softmax-attention GAT forward + backward on its rows of the global inputs,
and writes the results -- or the errors raised -- to <outdir>/<case>_rank<r>.npz.

Transports as in tests/mp_worker.py: "gloo" (ranks sharing one GPU), "nccl" (one GPU per rank)."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests.mp_gat_backward_worker import output_grad  # noqa: E402
from tests.mp_worker import gat_inputs, gather_local, sval  # noqa: E402


def score(r, c):
    """The edge scores of a case: up to +-1000, a function of the global coordinate."""
    r, c = np.asarray(r, np.float64), np.asarray(c, np.float64)
    return 1000.0 * np.sin(0.37 * r + 1.91 * c) * np.cos(0.11 * c)


def masked(r, c, N):
    """The entries a masked case scores -inf: in every fifth row each entry in the first half of the columns, in the
    next row every entry of an even column."""
    r, c = np.asarray(r), np.asarray(c)
    return ((r % 5 == 0) & (c < N // 2)) | ((r % 5 == 1) & (c % 2 == 0))


def upstream(r, c):
    """dL/d alpha of a case."""
    return np.cos(0.5 * np.asarray(r, np.float64) - 0.3 * np.asarray(c, np.float64))


def coords(alg, mode):
    """(row, col) of every entry of this rank's value vector of `mode`: SDDMMs of a global-index column against ones."""
    d = alg.dims
    A, B = alg.like_A_matrix(), alg.like_B_matrix()
    like = alg.like_S_values if mode == "A" else alg.like_ST_values
    sddmm = alg.sddmmA if mode == "A" else alg.sddmmB
    ones, res = like(1.0), like(0.0)
    out = []
    for first in ("A", "B"):
        for m, which, shape in ((A, "A", (d.localArows, d.localAcols)), (B, "B", (d.localBrows, d.localBcols))):
            top, _, nr, _ = alg.submatrices(which)[0]
            x = np.zeros(shape)
            x[:nr, 0] = np.arange(top, top + nr) if which == first else 1.0
            m.from_host(x)
        alg.initial_shift(A, B, "sddmm" + mode)
        sddmm(A, B, ones, res)
        alg.de_shift(A, B, "sddmm" + mode)
        out.append(np.rint(res.to_host()).astype(np.int64))
    return out


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
        per = N // world
        tr, tc, _ = orc.er_tuples(logM, npr, seed, per * rank, N if rank == world - 1 else per * (rank + 1))
        S = D.SpmatLocal.from_tuples(N, N, tr, tc, sval(tr, tc))
        layers, X0, weights = gat_inputs(N, case["layers"], seed)
        alg = D.Algorithm(alg_name, S, layers[0][0], c)
        out = {}
        if case.get("rejected"):
            # a layout without a row softmax: both entry points must refuse before any launch
            net = D.GAT(alg, layers, case["alpha"], attention="softmax")
            for key, call in (("softmax_error", lambda: alg.edge_softmax(alg.like_S_values(0.0), "A")),
                              ("gat_error", net.forward)):
                try:
                    call()
                except RuntimeError as e:
                    out[key] = str(e)
            np.savez(os.path.join(outdir, f"{name}_rank{rank}.npz"), **out)
            del net, alg, S
            continue
        # edge softmax in both orders
        try:
            for mode in ("A", "B"):
                r, cc = coords(alg, mode)
                like = alg.like_S_values if mode == "A" else alg.like_ST_values
                v, g = like(0.0), like(0.0)
                x = score(r, cc)
                if case.get("mask"):
                    x[masked(r, cc, N)] = -np.inf
                v.from_host(x)
                alg.edge_softmax(v, mode)
                a = v.to_host()
                g.from_host(upstream(r, cc))
                alg.edge_softmax_backward(v, g, mode)
                out.update({f"{mode}_rows": r, f"{mode}_cols": cc, f"{mode}_alpha": a, f"{mode}_dx": g.to_host()})
        except RuntimeError as e:
            out["softmax_error"] = str(e)
        if case.get("mask"):  # the masked case checks the edge softmax only
            np.savez(os.path.join(outdir, f"{name}_rank{rank}.npz"), **out)
            del alg, S
            continue
        # softmax-attention GAT: this rank's rows of the global input, the global weights and output gradient
        net = D.GAT(alg, layers, case["alpha"], attention="softmax")
        topB, _, nrB, _ = alg.submatrices("B")[0]
        topA, _, nrA, _ = alg.submatrices("A")[0]
        out.update(topA=topA, nrA=nrA, topB=topB, nrB=nrB)
        for i, (_, _, heads) in enumerate(layers):
            for h in range(heads):
                net.set_weight(i, h, weights[i][h])
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
        except RuntimeError as e:
            out["gat_error"] = str(e)
        np.savez(os.path.join(outdir, f"{name}_rank{rank}.npz"), **out)
        del net, alg, S
    D.world_finalize()


if __name__ == "__main__":
    main()
