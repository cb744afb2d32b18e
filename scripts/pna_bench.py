#!/usr/bin/env python
"""PNA on one GPU: the multi-statistic aggregation kernels against the four single-statistic passes they replace, and
the PNA train step beside GraphSAGE-mean's.  Prints the card name and power limit first, then one JSON line per
measurement.

kernels (an Erdos-Renyi 2^LOGM x 2^LOGM block with NPR draws per row, f in FS, normal inputs, REPS launches between
CUDA events):
  - forward: hnh_multi_aggregate_step_f64 with every statistic, against the composed baseline on the same block:
    hnh_spmm_f64 on Z and on Z^2, hnh_max_aggregate_step_f64 on Z and on -Z (preparing Z^2 and -Z is not timed);
  - backward: hnh_multi_aggregate_grad_f64 against hnh_spmm_f64 twice and hnh_max_aggregate_grad_f64 twice;
  - the share of 3.35 TB/s on each fused kernel's minimal bytes:
        forward   nnz (8 + 8 f) + rows (8 + 96 f)   (col_idx, the gathered rows; rowStart, six windows read and written)
        backward  nnz (8 + 48 f) + rows (8 + 24 f)  (col_idx, six gathered windows; rowStart, X, dX read and written)
train (2^TRAIN_LOGM nodes, NPR draws per row, GraphSAGE's bench widths 256 -> 1024 -> 1024 -> 1536, 15d_fusion1 at
  p = 1): the median of TRIALS train_step calls of PNA with [mean, min, max, std] x [identity, amplification,
  attenuation] and of GraphSAGE-mean, and PNA's graph_train_step (mean readout, 64 graphs, a 10-class head) beside its
  train_step.  PNA keeps P, (A S + 1) f doubles per row per layer, so TRAIN_LOGM defaults to 16: at 18 those widths
  need more than 80 GB.

Environment: PARTS (kernels,train), LOGM (20), NPR (32), FS (64,128,256), REPS (20), TRAIN_LOGM (16), TRIALS (3)."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM = 3.35e12
SAGE_LAYERS = [(256, 1024), (1024, 1024), (1024, 1536)]


def env(name, default):
    return os.environ.get(name, default)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def forward_bytes(nnz, rows, f):
    return nnz * (8 + 8 * f) + rows * (8 + 96 * f)


def backward_bytes(nnz, rows, f):
    return nnz * (8 + 48 * f) + rows * (8 + 24 * f)


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
    vals = torch.ones(len(col), dtype=torch.float64, device="cuda")
    nnz = len(col)
    del rows_g, cols_g, vals_g, order
    st = torch.cuda.current_stream().cuda_stream
    L = lib()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    rs, ci = rowStart.data_ptr(), col.data_ptr()

    def kern(fns):
        for fn in fns:
            fn()
        ev[0].record()
        for _ in range(reps):
            for fn in fns:
                fn()
        ev[1].record()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]) / 1e3 / reps

    for f in [int(x) for x in env("FS", "64,128,256").split(",")]:
        gen = torch.Generator(device="cuda").manual_seed(f)
        Z = torch.randn((n, f), dtype=torch.float64, device="cuda", generator=gen)
        Z2, Zn = Z * Z, -Z
        A = torch.zeros((n, 6 * f), dtype=torch.float64, device="cuda")
        check(L.hnh_multi_aggregate_step_f64(rs, ci, n, nnz, Z.data_ptr(), f, f, 7, A.data_ptr(), 6 * f, st), "multi_aggregate_step")
        check(L.hnh_multi_aggregate_finish_f64(A.data_ptr(), 6 * f, n, f, 7, st), "multi_aggregate_finish")
        Dm = torch.empty_like(A)
        dA = torch.randn((n, 6 * f), dtype=torch.float64, device="cuda", generator=gen)
        check(L.hnh_multi_aggregate_grad_prep_f64(A.data_ptr(), 6 * f, dA.data_ptr(), 6 * f, n, f, 7, Dm.data_ptr(), 6 * f, st), "prep")
        del dA
        Y1, Y2, M1, C1, M2, C2 = (torch.zeros((n, f), dtype=torch.float64, device="cuda") for _ in range(6))
        G1, G2, dX = (torch.rand((n, f), dtype=torch.float64, device="cuda", generator=gen) for _ in range(3))
        fwd = kern([lambda: L.hnh_multi_aggregate_step_f64(rs, ci, n, nnz, Z.data_ptr(), f, f, 7, A.data_ptr(), 6 * f, st)])
        composed_fwd = kern([
            lambda: L.hnh_spmm_f64(rs, ci, vals.data_ptr(), n, nnz, Z.data_ptr(), Y1.data_ptr(), f, 0, st),
            lambda: L.hnh_spmm_f64(rs, ci, vals.data_ptr(), n, nnz, Z2.data_ptr(), Y2.data_ptr(), f, 0, st),
            lambda: L.hnh_max_aggregate_step_f64(rs, ci, n, nnz, Z.data_ptr(), f, f, M1.data_ptr(), f, C1.data_ptr(), f, st),
            lambda: L.hnh_max_aggregate_step_f64(rs, ci, n, nnz, Zn.data_ptr(), f, f, M2.data_ptr(), f, C2.data_ptr(), f, st)])
        bwd = kern([lambda: L.hnh_multi_aggregate_grad_f64(rs, ci, n, nnz, Z.data_ptr(), f, Dm.data_ptr(), 6 * f, f, 7, dX.data_ptr(), f,
                                                           st)])
        composed_bwd = kern([
            lambda: L.hnh_spmm_f64(rs, ci, vals.data_ptr(), n, nnz, G1.data_ptr(), dX.data_ptr(), f, 0, st),
            lambda: L.hnh_spmm_f64(rs, ci, vals.data_ptr(), n, nnz, G2.data_ptr(), dX.data_ptr(), f, 0, st),
            lambda: L.hnh_max_aggregate_grad_f64(rs, ci, n, nnz, Z.data_ptr(), f, M1.data_ptr(), f, G1.data_ptr(), f, f, dX.data_ptr(), f,
                                                 st),
            lambda: L.hnh_max_aggregate_grad_f64(rs, ci, n, nnz, Zn.data_ptr(), f, M2.data_ptr(), f, G2.data_ptr(), f, f,
                                                 dX.data_ptr(), f, st)])
        out(dict(part="kernels", f=f, n=n, nnz=nnz, forward_ms=fwd * 1e3, composed_forward_ms=composed_fwd * 1e3,
                 forward_over_composed=fwd / composed_fwd, forward_hbm_share=forward_bytes(nnz, n, f) / fwd / HBM,
                 backward_ms=bwd * 1e3, composed_backward_ms=composed_bwd * 1e3, backward_over_composed=bwd / composed_bwd,
                 backward_hbm_share=backward_bytes(nnz, n, f) / bwd / HBM))
        del Z, Z2, Zn, A, Dm, Y1, Y2, M1, C1, M2, C2, G1, G2, dX
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
    logM, npr, trials = int(env("TRAIN_LOGM", "16")), int(env("NPR", "32")), int(env("TRIALS", "3"))
    S = D.SpmatLocal.load_er(logM, npr, 0xC0FFEE)
    rows_g = S.tuples()[0]
    hist = np.bincount(np.bincount(np.asarray(rows_g, np.int64), minlength=1 << logM))
    rng = np.random.default_rng(3)
    for model in ("pna", "sage_mean"):
        alg = D.Algorithm("15d_fusion1", S, SAGE_LAYERS[0][0], 1)
        net = D.PNA(alg, SAGE_LAYERS, deg=hist) if model == "pna" else D.GraphSAGE(alg, SAGE_LAYERS, aggr="mean")
        classes = SAGE_LAYERS[-1][1]
        for l in range(len(net.layers)):
            for name in net.param_names():
                s = net.param_shape(l, name)
                net.set_param(l, name, rng.uniform(-1, 1, s) * (0.05 if len(s) == 1 else 1 / np.sqrt(s[0])))
        net.set_input(rng.uniform(-1, 1, net.buffer_shape(0)))
        last = len(net.layers)
        rows_local = net.buffer_shape(last)[0]
        lab = rng.integers(0, classes, rows_local)
        lab[1 << logM:] = -1
        labels = D.NodeLabels(net, lab, classes)
        opt = D.AdamW(lr=1e-3)
        net.train_step(labels, opt)
        t = [timed(lambda: net.train_step(labels, opt)) for _ in range(trials)]
        out(dict(part="train_step", model=model, logM=logM, nnz_per_row=npr, s_per_call=round(float(np.median(t)), 4)))
        if model == "pna":
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
