#!/usr/bin/env python
"""GIN and GINE on one GPU: the three edge-ReLU aggregation kernels against the torch composition they replace, and the
GIN / GINE train steps beside GraphSAGE-sum's.  Prints the card name and power limit first, then one JSON line per
measurement.

kernels (an Erdos-Renyi 2^LOGM x 2^LOGM block with NPR draws per row, f in FS, normal inputs, REPS launches between
CUDA events after one warm-up launch each):
  - hnh_edge_relu_aggregate_step_f64 (forward, A order), hnh_edge_relu_aggregate_grad_f64 (dX, on the transposed
    block with E in its order) and hnh_edge_relu_aggregate_edge_grad_f64 (dE, A order);
  - the share of 3.35 TB/s on each kernel's minimal bytes:
        forward  nnz (8 + 16 f) + rows (8 + 16 f)   (col_idx, the gathered X row, E_i; rowStart, A read and written)
        dX       nnz (8 + 16 f) + rows (8 + 24 f)   (col_idx, the gathered dA row, E_i; rowStart, X, dX read and written)
        dE       nnz (8 + 24 f) + rows (8 + 8 f)    (col_idx, the gathered X row, E_i, dE_i written; rowStart, dA)
  - the baseline: the torch composition on the same device in fp64, timed the same way: forward
    index_select(X, cols) + E, relu, index_add_ over the rows; backward index_select(dA, rows) masked by
    index_select(X, cols) + E > 0 (that is dE), then index_add_ of it over the columns (dX).  It materialises the
    nnz x f messages the kernels never hold.
train (2^TRAIN_LOGM nodes, NPR draws per row, 15d_fusion1 at p = 1; OGB-like widths: 5 layers (300, 600, 300), edge_dim
  8): the median of TRIALS train_step calls of GIN, GINE and GraphSAGE-sum (5 layers 300 -> 300), and GINE's
  graph_train_step (mean readout, 64 graphs, a 10-class head) beside its train_step.  A GINE backward holds E_A, E_B
  and dE_A, 3 nnz f doubles: TRAIN_LOGM defaults to 17 (10 GB each at NPR = 32).

Environment: PARTS (kernels,train), LOGM (20), NPR (32), FS (32,64), REPS (20), TRAIN_LOGM (17), TRIALS (3)."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM = 3.35e12
GIN_LAYERS = [(300, 600, 300)] * 5
SAGE_LAYERS = [(300, 300)] * 5
EDGE_DIM = 8


def env(name, default):
    return os.environ.get(name, default)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def forward_bytes(nnz, rows, f):
    return nnz * (8 + 16 * f) + rows * (8 + 16 * f)


def grad_bytes(nnz, rows, f):
    return nnz * (8 + 16 * f) + rows * (8 + 24 * f)


def edge_grad_bytes(nnz, rows, f):
    return nnz * (8 + 24 * f) + rows * (8 + 8 * f)


def kernels_part(out):
    import numpy as np
    import torch

    from distributed_sddmm_b200 import check, lib
    from distributed_sddmm_b200 import driver as D
    logM, npr, reps = int(env("LOGM", "20")), int(env("NPR", "32")), int(env("REPS", "20"))
    S = D.SpmatLocal.load_er(logM, npr, 0xC0FFEE)
    rows_g, cols_g, _ = S.tuples()
    rows_g, cols_g = np.asarray(rows_g, np.int64), np.asarray(cols_g, np.int64)
    order = np.lexsort((cols_g, rows_g))
    rows_g, cols_g = rows_g[order], cols_g[order]
    n = 1 << logM
    nnz = len(cols_g)
    rowStart = torch.from_numpy(np.searchsorted(rows_g, np.arange(n + 1)).astype(np.int64)).cuda()
    col, row = torch.from_numpy(cols_g).cuda(), torch.from_numpy(rows_g).cuda()
    # the transposed block: its entry k is entry perm[k] of the A order
    perm_h = np.lexsort((rows_g, cols_g))
    tStart = torch.from_numpy(np.searchsorted(cols_g[perm_h], np.arange(n + 1)).astype(np.int64)).cuda()
    tcol, perm = torch.from_numpy(rows_g[perm_h]).cuda(), torch.from_numpy(perm_h.astype(np.int64)).cuda()
    del rows_g, cols_g, order, perm_h
    st = torch.cuda.current_stream().cuda_stream
    L = lib()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def kern(fn):
        fn()
        ev[0].record()
        for _ in range(reps):
            fn()
        ev[1].record()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]) / 1e3 / reps

    for f in [int(x) for x in env("FS", "32,64").split(",")]:
        gen = torch.Generator(device="cuda").manual_seed(f)
        X = torch.randn((n, f), dtype=torch.float64, device="cuda", generator=gen)
        dA = torch.randn((n, f), dtype=torch.float64, device="cuda", generator=gen)
        E = torch.randn((nnz, f), dtype=torch.float64, device="cuda", generator=gen)
        A, dX = torch.zeros((n, f), dtype=torch.float64, device="cuda"), torch.zeros((n, f), dtype=torch.float64, device="cuda")
        rs, ci = rowStart.data_ptr(), col.data_ptr()
        fwd = kern(lambda: check(L.hnh_edge_relu_aggregate_step_f64(rs, ci, n, nnz, X.data_ptr(), f, E.data_ptr(), f, f, A.data_ptr(),
                                                                    f, st), "edge_relu_aggregate_step"))
        dE = torch.empty_like(E)
        egrad = kern(lambda: check(L.hnh_edge_relu_aggregate_edge_grad_f64(rs, ci, n, nnz, dA.data_ptr(), f, X.data_ptr(), f,
                                                                           E.data_ptr(), f, f, dE.data_ptr(), f, st),
                                   "edge_relu_aggregate_edge_grad"))
        del dE
        EB = E.index_select(0, perm)
        grad = kern(lambda: check(L.hnh_edge_relu_aggregate_grad_f64(tStart.data_ptr(), tcol.data_ptr(), n, nnz, X.data_ptr(), f,
                                                                     EB.data_ptr(), f, dA.data_ptr(), f, f, dX.data_ptr(), f, st),
                                  "edge_relu_aggregate_grad"))
        del EB
        torch.cuda.empty_cache()

        def torch_forward():
            msg = X.index_select(0, col)
            msg.add_(E).relu_()
            A.zero_().index_add_(0, row, msg)

        def torch_backward():
            g = dA.index_select(0, row)
            s = X.index_select(0, col)
            g.mul_(s.add_(E) > 0)  # dE
            del s
            dX.zero_().index_add_(0, col, g)

        tf, tb = kern(torch_forward), kern(torch_backward)
        fused = fwd + grad + egrad
        out(dict(part="kernels", f=f, n=n, nnz=nnz, forward_ms=fwd * 1e3, forward_hbm_share=forward_bytes(nnz, n, f) / fwd / HBM,
                 grad_ms=grad * 1e3, grad_hbm_share=grad_bytes(nnz, n, f) / grad / HBM, edge_grad_ms=egrad * 1e3,
                 edge_grad_hbm_share=edge_grad_bytes(nnz, n, f) / egrad / HBM, torch_forward_ms=tf * 1e3, torch_backward_ms=tb * 1e3,
                 fused_total_ms=fused * 1e3, torch_total_ms=(tf + tb) * 1e3, torch_over_fused=(tf + tb) / fused))
        del X, dA, E, A, dX
        torch.cuda.empty_cache()


def timed(fn):
    """Seconds of one call between CUDA events on the current stream (the library's streams are ordered after it)."""
    import torch
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    torch.cuda.synchronize()
    ev[0].record()
    fn()
    torch.cuda.synchronize()
    ev[1].record()
    ev[1].synchronize()
    return ev[0].elapsed_time(ev[1]) / 1e3


def train_part(out):
    import numpy as np
    import torch

    from distributed_sddmm_b200 import driver as D
    logM, npr, trials = int(env("TRAIN_LOGM", "17")), int(env("NPR", "32")), int(env("TRIALS", "3"))
    S = D.SpmatLocal.load_er(logM, npr, 0xC0FFEE)
    rng = np.random.default_rng(3)
    classes = GIN_LAYERS[-1][2]  # node labels over the output width, as pna_bench.py
    for model in ("gin", "gine", "sage_sum"):
        alg = D.Algorithm("15d_fusion1", S, GIN_LAYERS[0][0], 1)
        if model == "sage_sum":
            net = D.GraphSAGE(alg, SAGE_LAYERS, aggr="sum")
        else:
            net = D.GIN(alg, GIN_LAYERS, edge_dim=EDGE_DIM if model == "gine" else 0, train_eps=True)
        for l in range(len(net.layers)):
            for name in net.param_names():
                s = net.param_shape(l, name)
                net.set_param(l, name, rng.uniform(-1, 1, s) * (0.05 if len(s) == 1 else 1 / np.sqrt(s[0])))
        if model == "gine":
            na, nb = len(alg.like_S_values()), len(alg.like_ST_values())
            net.set_edge_attributes(rng.uniform(-1, 1, (na, EDGE_DIM)), rng.uniform(-1, 1, (nb, EDGE_DIM)))
        net.set_input(rng.uniform(-1, 1, net.buffer_shape(0)))
        rows_local = net.buffer_shape(len(net.layers))[0]
        lab = rng.integers(0, classes, rows_local)
        lab[1 << logM:] = -1
        labels = D.NodeLabels(net, lab, classes)
        opt = D.AdamW(lr=1e-3)
        net.train_step(labels, opt)
        t = [timed(lambda: net.train_step(labels, opt)) for _ in range(trials)]
        out(dict(part="train_step", model=model, logM=logM, nnz_per_row=npr, s_per_call=round(float(np.median(t)), 4)))
        if model == "gine":
            G = 64
            batch = np.full(rows_local, -1, np.int64)
            batch[:1 << logM] = np.sort(rng.integers(0, G, 1 << logM))
            ro = D.GraphReadout(net, batch, G, pool="mean", num_classes=10)
            gl = D.GraphLabels(ro, rng.integers(0, 10, G), 10)
            gopt = D.AdamW(lr=1e-3)  # the head adds parameters: an optimizer of its own
            net.graph_train_step(ro, gl, gopt)
            tg = [timed(lambda: net.graph_train_step(ro, gl, gopt)) for _ in range(trials)]
            out(dict(part="graph_train_step", model=model, logM=logM, graphs=G, s_per_call=round(float(np.median(tg)), 4),
                     over_train_step=float(np.median(tg)) / float(np.median(t))))
            del ro, gl, gopt
        del net, labels, opt, alg
        torch.cuda.empty_cache()


def main():
    import torch

    from distributed_sddmm_b200 import driver as D
    print(json.dumps(dict(card=card())), flush=True)
    torch.cuda.set_device(0)
    D.world_init("self")
    out = lambda rec: print(json.dumps(rec), flush=True)  # noqa: E731
    parts = env("PARTS", "kernels,train").split(",")
    if "kernels" in parts:
        kernels_part(out)
    if "train" in parts:
        train_part(out)
    D.world_finalize()


if __name__ == "__main__":
    main()
