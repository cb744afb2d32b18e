#!/usr/bin/env python
"""GraphSAGE on one GPU: the max-aggregation kernels against the accumulating SpMM kernel, and the SAGE train step beside
the graph transformer's.  Prints the card name and power limit first, then one JSON line per measurement.

kernels (an Erdos-Renyi 2^LOGM x 2^LOGM block with NPR draws per row, f in FS, inputs "normal" or "relu" (half zeros),
REPS launches between CUDA events):
  - step: hnh_max_aggregate_step_f64 into [Z | C]; spmm: hnh_spmm_f64 accumulating into Y on the same block and X;
    grad: hnh_max_aggregate_grad_f64 with the step's Z and G = 1 / C;
  - the share of 3.35 TB/s on each kernel's algorithmic bytes:
        step   nnz (8 + 8 f) + rows (8 + 32 f)     (col_idx, the gathered rows; rowStart, [Z | C] read and written)
        grad   nnz (8 + 16 f) + rows (8 + 24 f)    (col_idx, the gathered [Z | G]; rowStart, X, dX read and written)
        spmm   nnz (16 + 8 f) + rows (8 + 16 f)    (col_idx and values, the gathered rows; rowStart, Y read and written)
train (2^TRAIN_LOGM nodes, NPR draws per row, the graph transformer bench's widths 256 -> 1024 -> 1024 -> 1536,
  15d_fusion1 at p = 1): the median of TRIALS train_step calls of GraphSAGE with each aggregator and of the graph
  transformer [(256, 256, 4), (1024, 256, 4), (1024, 256, 6)].

Environment: PARTS (kernels,train), LOGM (20), NPR (32), FS (64,128,256), REPS (20), TRAIN_LOGM (18), TRIALS (3)."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM = 3.35e12
SAGE_LAYERS = [(256, 1024), (1024, 1024), (1024, 1536)]
GT_LAYERS = [(256, 256, 4), (1024, 256, 4), (1024, 256, 6)]


def env(name, default):
    return os.environ.get(name, default)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def step_bytes(nnz, rows, f):
    return nnz * (8 + 8 * f) + rows * (8 + 32 * f)


def grad_bytes(nnz, rows, f):
    return nnz * (8 + 16 * f) + rows * (8 + 24 * f)


def spmm_bytes(nnz, rows, f):
    return nnz * (16 + 8 * f) + rows * (8 + 16 * f)


def kernels_part(out):
    import numpy as np
    import torch

    from distributed_sddmm_b200 import check, lib
    from distributed_sddmm_b200 import driver as D
    logM, npr, reps = int(env("LOGM", "20")), int(env("NPR", "32")), int(env("REPS", "20"))
    S = D.SpmatLocal.load_er(logM, npr, 0xC0FFEE)
    rows_g, cols_g, vals_g = S.tuples()
    order = np.lexsort((cols_g, rows_g))
    n = 1 << logM
    rowStart = torch.from_numpy(np.searchsorted(rows_g[order], np.arange(n + 1)).astype(np.int64)).cuda()
    col = torch.from_numpy(cols_g[order].astype(np.int64)).cuda()
    vals = torch.from_numpy(vals_g[order]).cuda()
    nnz = len(col)
    del rows_g, cols_g, vals_g, order
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

    for f in [int(x) for x in env("FS", "64,128,256").split(",")]:
        for kind in ("normal", "relu"):
            gen = torch.Generator(device="cuda").manual_seed(f)
            X = torch.randn((n, f), dtype=torch.float64, device="cuda", generator=gen)
            if kind == "relu":
                X.clamp_(min=0.0)
            Z = torch.full((n, f), -np.inf, dtype=torch.float64, device="cuda")
            Cn = torch.zeros((n, f), dtype=torch.float64, device="cuda")
            Y, dX = torch.zeros_like(X), torch.zeros_like(X)
            check(L.hnh_max_aggregate_step_f64(rowStart.data_ptr(), col.data_ptr(), n, nnz, X.data_ptr(), f, f, Z.data_ptr(), f,
                                               Cn.data_ptr(), f, st), "max_aggregate_step")
            check(L.hnh_max_aggregate_finish_f64(Z.data_ptr(), Cn.data_ptr(), n * f, st), "max_aggregate_finish")
            G = torch.where(Cn > 0, 1.0 / Cn.clamp(min=1.0), torch.zeros_like(Cn))
            ties = float((Cn > 1).double().mean())
            t_step = kern(lambda: L.hnh_max_aggregate_step_f64(rowStart.data_ptr(), col.data_ptr(), n, nnz, X.data_ptr(), f, f,
                                                               Z.data_ptr(), f, Cn.data_ptr(), f, st))
            t_grad = kern(lambda: L.hnh_max_aggregate_grad_f64(rowStart.data_ptr(), col.data_ptr(), n, nnz, X.data_ptr(), f,
                                                               Z.data_ptr(), f, G.data_ptr(), f, f, dX.data_ptr(), f, st))
            t_spmm = kern(lambda: L.hnh_spmm_f64(rowStart.data_ptr(), col.data_ptr(), vals.data_ptr(), n, nnz, X.data_ptr(),
                                                 Y.data_ptr(), f, 0, st))
            out(dict(part="kernels", f=f, inputs=kind, n=n, nnz=nnz, tied_share=round(ties, 4), step_ms=t_step * 1e3,
                     grad_ms=t_grad * 1e3, spmm_ms=t_spmm * 1e3, step_over_spmm=t_step / t_spmm,
                     step_hbm_share=step_bytes(nnz, n, f) / t_step / HBM, grad_hbm_share=grad_bytes(nnz, n, f) / t_grad / HBM,
                     spmm_hbm_share=spmm_bytes(nnz, n, f) / t_spmm / HBM))
            del X, Z, Cn, Y, dX, G


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def train_part(out):
    import numpy as np

    from distributed_sddmm_b200 import driver as D
    logM, npr, trials = int(env("TRAIN_LOGM", "18")), int(env("NPR", "32")), int(env("TRIALS", "3"))
    S = D.SpmatLocal.load_er(logM, npr, 0xC0FFEE)
    rng = np.random.default_rng(3)
    for model in ("sage_mean", "sage_sum", "sage_max", "graph_transformer"):
        alg = D.Algorithm("15d_fusion1", S, SAGE_LAYERS[0][0], 1)
        if model == "graph_transformer":
            net, classes = D.GraphTransformer(alg, GT_LAYERS), GT_LAYERS[-1][1] * GT_LAYERS[-1][2]
        else:
            net, classes = D.GraphSAGE(alg, SAGE_LAYERS, aggr=model[5:]), SAGE_LAYERS[-1][1]
        for l in range(len(net.layers)):
            for name in net.param_names():
                s = net.param_shape(l, name)
                net.set_param(l, name, rng.uniform(-1, 1, s) * (0.05 if len(s) == 1 else 1 / np.sqrt(s[0])))
        net.set_input(rng.uniform(-1, 1, net.buffer_shape(0)))
        last = len(net.layers)
        lab = rng.integers(0, classes, net.buffer_shape(last)[0])
        lab[1 << logM:] = -1
        labels = D.NodeLabels(net, lab, classes)
        opt = D.AdamW(lr=1e-3)
        net.train_step(labels, opt)
        t = [timed(lambda: net.train_step(labels, opt)) for _ in range(trials)]
        out(dict(part="train_step", model=model, logM=logM, nnz_per_row=npr, s_per_call=round(float(np.median(t)), 4)))
        del net, labels, opt, alg


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
