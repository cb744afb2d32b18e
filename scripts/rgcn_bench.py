#!/usr/bin/env python
"""R-GCN on one GPU: the relational-aggregation kernels against the accumulating SpMM kernel, and the R-GCN train step
beside GraphSAGE's mean.  Prints the card name and power limit first, then one JSON line per measurement.

kernels (an Erdos-Renyi 2^LOGM x 2^LOGM block with NPR draws per row, relations uniform at random in [0, R) for R in RS,
f in FS, REPS launches between CUDA events):
  - step: hnh_relational_aggregate_f64 adding into A (R f wide); zero: hnh_fill_f64 of A, which the op runs before the
    first block; grad: hnh_relational_aggregate_grad_f64 adding into dX with A as dA; spmm: hnh_spmm_f64 accumulating
    into Y on the same block and X;
  - the share of 3.35 TB/s on each kernel's algorithmic bytes:
        step   nnz (16 + 8 f) + (rows + 1) 8 + 16 f W   (col_idx and value, the gathered rows; rowStart; each of the W
                                                        distinct (stored row, relation) windows read and written once)
        grad   nnz (16 + 8 f) + (rows + 1) 8 + 16 rows f   (the accumulating SpMM's bytes, the relation in place of the
                                                        weight)
        spmm   the same as grad
        zero   8 rows R f
    W is counted on the host from the tuples.
train (2^TRAIN_LOGM nodes, NPR draws per row, GraphSAGE's bench widths 256 -> 1024 -> 1024 -> 1536, 15d_fusion1 at
  p = 1): the median of TRIALS train_step calls of R-GCN (mean and sum, R = TRAIN_R relations uniform at random) and of
  GraphSAGE with the mean.  At R = 4 an R-GCN layer of input width 1024 keeps 2^18 x 4096 doubles (8.6 GB).

Environment: PARTS (kernels,train), LOGM (20), NPR (32), FS (64,128,256), RS (4,8), REPS (20), TRAIN_LOGM (18),
TRAIN_R (4), TRIALS (3)."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM = 3.35e12
LAYERS = [(256, 1024), (1024, 1024), (1024, 1536)]


def env(name, default):
    return os.environ.get(name, default)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def step_bytes(nnz, rows, f, W):
    return nnz * (16 + 8 * f) + (rows + 1) * 8 + 16 * f * W


def grad_bytes(nnz, rows, f):
    return nnz * (16 + 8 * f) + (rows + 1) * 8 + 16 * rows * f


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
    rows_s = rows_g[order].astype(np.int64)
    rowStart = torch.from_numpy(np.searchsorted(rows_s, np.arange(n + 1)).astype(np.int64)).cuda()
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

    rng = np.random.default_rng(5)
    for R in [int(x) for x in env("RS", "4,8").split(",")]:
        rel_h = rng.integers(0, R, nnz)
        W = len(np.unique(rows_s * R + rel_h))
        rel = torch.from_numpy(rel_h.astype(np.float64)).cuda()
        for f in [int(x) for x in env("FS", "64,128,256").split(",")]:
            gen = torch.Generator(device="cuda").manual_seed(f)
            X = torch.randn((n, f), dtype=torch.float64, device="cuda", generator=gen)
            A = torch.zeros((n, R * f), dtype=torch.float64, device="cuda")
            Y, dX = torch.zeros_like(X), torch.zeros_like(X)
            t_zero = kern(lambda: L.hnh_fill_f64(A.data_ptr(), n * R * f, 0.0, st))
            check(L.hnh_relational_aggregate_f64(rowStart.data_ptr(), col.data_ptr(), rel.data_ptr(), n, nnz, X.data_ptr(), f, f, R,
                                                 A.data_ptr(), R * f, st), "relational_aggregate")
            t_step = kern(lambda: L.hnh_relational_aggregate_f64(rowStart.data_ptr(), col.data_ptr(), rel.data_ptr(), n, nnz,
                                                                 X.data_ptr(), f, f, R, A.data_ptr(), R * f, st))
            t_grad = kern(lambda: L.hnh_relational_aggregate_grad_f64(rowStart.data_ptr(), col.data_ptr(), rel.data_ptr(), n, nnz,
                                                                      A.data_ptr(), R * f, f, R, dX.data_ptr(), f, st))
            t_spmm = kern(lambda: L.hnh_spmm_f64(rowStart.data_ptr(), col.data_ptr(), vals.data_ptr(), n, nnz, X.data_ptr(),
                                                 Y.data_ptr(), f, 0, st))
            out(dict(part="kernels", R=R, f=f, n=n, nnz=nnz, windows=W, zero_ms=t_zero * 1e3, step_ms=t_step * 1e3,
                     grad_ms=t_grad * 1e3, spmm_ms=t_spmm * 1e3, step_over_spmm=t_step / t_spmm, grad_over_spmm=t_grad / t_spmm,
                     step_hbm_share=step_bytes(nnz, n, f, W) / t_step / HBM, grad_hbm_share=grad_bytes(nnz, n, f) / t_grad / HBM,
                     spmm_hbm_share=grad_bytes(nnz, n, f) / t_spmm / HBM, zero_hbm_share=8 * n * R * f / t_zero / HBM))
            del X, A, Y, dX


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
    logM, npr, trials, R = int(env("TRAIN_LOGM", "18")), int(env("NPR", "32")), int(env("TRIALS", "3")), int(env("TRAIN_R", "4"))
    S0 = D.SpmatLocal.load_er(logM, npr, 0xC0FFEE)
    rows, cols, _ = S0.tuples()
    rng = np.random.default_rng(3)
    S = D.SpmatLocal.from_tuples(1 << logM, 1 << logM, rows, cols, rng.integers(0, R, len(rows)).astype(np.float64))
    del S0
    for model in ("rgcn_mean", "rgcn_sum", "sage_mean"):
        alg = D.Algorithm("15d_fusion1", S, LAYERS[0][0], 1)
        if model.startswith("rgcn"):
            net = D.RGCN(alg, LAYERS, num_relations=R, aggr=model[5:])
        else:
            net = D.GraphSAGE(alg, LAYERS, aggr="mean")
        classes = LAYERS[-1][1]
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
        out(dict(part="train_step", model=model, relations=R if model.startswith("rgcn") else 1, logM=logM, nnz_per_row=npr,
                 s_per_call=round(float(np.median(t)), 4)))
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
