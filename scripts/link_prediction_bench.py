#!/usr/bin/env python
"""Link prediction on one GPU: the fused edge decoder against the flagship FusedMM kernel and against the composed
public-op path.  Prints the card name and power limit first, then one JSON line per measurement.

op (an Erdos-Renyi 2^LOGM x 2^LOGM target matrix T with NPR draws per row, targets 1, under 15d_fusion1 at p = 1, r in
RS; H random, H_A = H_B = H, dH_A = dH_B):
  - link_fwd / link_grad: Algorithm.link_loss without / with the gradient (1 / 2 gather passes, a sync each);
  - kernel_link / kernel_fused: hnh_link_bce_f64 with dX and stats (one pass) and hnh_fused_f64 (the flagship SDDMM ->
    SpMM row kernel) on the same CSR block and operands, REPS launches between CUDA events; the share of 3.35 TB/s on
    each pass's minimal bytes: the row side read once and its gradient read and written (3 n r 8), every gathered row
    (nnz r 8), col_idx and the values (nnz 16), rowStart (n 8), plus for link the stats (n 16 read and written);
  - composed: sddmmA and sddmmB of the scores, their download, the sigmoid gradient on the host, the upload, spmmA and
    spmmB, and the two halves downloaded and summed -- what a user can write from the public ops;
  - build: a fresh T (load_er with a new seed), its Algorithm and the LinkTargets of a model: the per-epoch cost of new
    negatives.
train (2^TRAIN_LOGM nodes, S and T Erdos-Renyi with NPR draws per row, a graph transformer with layers LAYERS): the
  median of TRIALS link_train_step calls against forward + backward from a host gradient of the same shape.

Environment: PARTS (op,train), LOGM (20), NPR (32), RS (64,128,256), REPS (10), TRIALS (5), TRAIN_LOGM (18)."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM = 3.35e12
LAYERS = [(128, 64, 2), (128, 128, 1)]


def env(name, default):
    return os.environ.get(name, default)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timed(fn, reps):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps


def op_part(out):
    import numpy as np
    import torch

    from distributed_sddmm_b200 import driver as D
    from distributed_sddmm_b200 import lib
    logM, npr, reps = int(env("LOGM", "20")), int(env("NPR", "32")), int(env("REPS", "10"))
    T = D.SpmatLocal.load_er(logM, npr, 0xC0FFEE)
    rows_g, cols_g, vals_g = T.tuples()
    order = np.lexsort((cols_g, rows_g))
    n = 1 << logM
    rowStart = torch.from_numpy(np.searchsorted(rows_g[order], np.arange(n + 1)).astype(np.int64)).cuda()
    col = torch.from_numpy(cols_g[order].astype(np.int64)).cuda()
    vals = torch.from_numpy(vals_g[order]).cuda()
    nnz = len(col)
    del rows_g, cols_g, vals_g, order
    st = torch.cuda.current_stream().cuda_stream
    for r in [int(x) for x in env("RS", "64,128,256").split(",")]:
        alg = D.Algorithm("15d_fusion1", T, r, 1)
        rows = alg.like_A_matrix().shape[0]
        rng = np.random.default_rng(r)
        Hh = rng.standard_normal((rows, r)) / np.sqrt(r)
        H, dH = D.Dense.create(rows, r), D.Dense.create(rows, r)
        H.from_host(Hh)
        alg.link_loss(H, H, dH, dH)
        fwd = timed(lambda: alg.link_loss(H, H), reps)
        grad = timed(lambda: alg.link_loss(H, H, dH, dH), reps)
        # the kernels alone, on the same CSR block
        X = torch.from_numpy(Hh[:n]).cuda()
        dX, Out = torch.zeros_like(X), torch.zeros_like(X)
        stats = torch.zeros((n, 2), dtype=torch.float64, device="cuda")
        v = vals.clone()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

        def kern(fn):
            fn()
            ev[0].record()
            for _ in range(reps):
                fn()
            ev[1].record()
            torch.cuda.synchronize()
            return ev[0].elapsed_time(ev[1]) / 1e3 / reps

        k_link = kern(lambda: lib().hnh_link_bce_f64(rowStart.data_ptr(), col.data_ptr(), vals.data_ptr(), n, nnz, X.data_ptr(), r,
                                                     X.data_ptr(), r, r, 1.0 / nnz, dX.data_ptr(), r, stats.data_ptr(), 2, None, st))
        k_fused = kern(lambda: lib().hnh_fused_f64(rowStart.data_ptr(), col.data_ptr(), v.data_ptr(), n, nnz, X.data_ptr(),
                                                   X.data_ptr(), Out.data_ptr(), r, 0, st))
        base = 3 * n * r * 8 + nnz * r * 8 + nnz * 16 + n * 8
        link_bytes, fused_bytes = base + 2 * n * 16, base
        # composed public-op path on its own algorithm object (the SDDMMs overwrite the block values)
        comp = D.Algorithm("15d_fusion1", T, r, 1)
        ones_A, ones_B = comp.like_S_values(1.0), comp.like_ST_values(1.0)
        sA, sB, gA, gB = comp.like_S_values(), comp.like_ST_values(), comp.like_S_values(), comp.like_ST_values()
        dA, dB = comp.like_A_matrix(), comp.like_B_matrix()

        def composed():
            comp.sddmmA(H, H, ones_A, sA)
            comp.sddmmB(H, H, ones_B, sB)
            for s, g in ((sA, gA), (sB, gB)):
                x = s.to_host()
                g.from_host((1.0 / (1.0 + np.exp(-x)) - 1.0) / nnz)
            comp.spmmA(dA, H, gA)
            comp.spmmB(H, dB, gB)
            return dA.to_host() + dB.to_host()  # a Dense has no device-side add among the public ops

        composed()
        t_comp = timed(composed, max(1, reps // 3))
        del comp, ones_A, ones_B, sA, sB, gA, gB, dA, dB
        rec = dict(part="op", r=r, n=n, nnz=nnz, link_fwd_ms=fwd * 1e3, link_grad_ms=grad * 1e3, kernel_link_ms=k_link * 1e3,
                   kernel_fused_ms=k_fused * 1e3, link_over_fused=k_link / k_fused,
                   link_hbm_share=link_bytes / k_link / HBM, fused_hbm_share=fused_bytes / k_fused / HBM,
                   fwd_pass_hbm_share=link_bytes / fwd / HBM, grad_hbm_share=2 * link_bytes / grad / HBM,
                   composed_ms=t_comp * 1e3, composed_over_grad=t_comp / grad)
        out(rec)
        del alg, H, dH, X, dX, Out, stats, v
    # the per-epoch cost of fresh targets
    model_alg = D.Algorithm("15d_fusion1", T, 64, 1)
    net = D.GraphTransformer(model_alg, [(64, 32, 2)])
    t0 = time.perf_counter()
    T2 = D.SpmatLocal.load_er(logM, npr, 0xBEEF)
    a2 = D.Algorithm("15d_fusion1", T2, 64, 1)
    D.LinkTargets(net, a2)
    out(dict(part="build", n=n, npr=npr, seconds=time.perf_counter() - t0))


def train_part(out):
    import numpy as np
    import torch

    from distributed_sddmm_b200 import driver as D
    logM, npr, trials = int(env("TRAIN_LOGM", "18")), int(env("NPR", "32")), int(env("TRIALS", "5"))
    S = D.SpmatLocal.load_er(logM, 16, 0xC0FFEE)
    alg = D.Algorithm("15d_fusion1", S, LAYERS[0][0], 1)
    net = D.GraphTransformer(alg, LAYERS)
    rng = np.random.default_rng(3)
    for l in range(len(LAYERS)):
        for name in net.param_names():
            s = net.param_shape(l, name)
            net.set_param(l, name, rng.uniform(-1, 1, s) * (0.05 if len(s) == 1 else 1 / np.sqrt(s[0])))
    net.set_input(rng.uniform(-1, 1, net.buffer_shape(0)))
    T = D.SpmatLocal.load_er(logM, npr, 0xBEEF)
    t = D.LinkTargets(net, D.Algorithm("15d_fusion1", T, LAYERS[0][0], 1))
    opt = D.AdamW(lr=1e-3)
    g = rng.standard_normal(net.buffer_shape(len(LAYERS)))
    net.link_train_step(t, opt)

    def fb():
        net.forward()
        net.backward(g)

    fb()
    step = [timed(lambda: net.link_train_step(t, opt), 1) for _ in range(trials)]
    ref = [timed(fb, 1) for _ in range(trials)]
    out(dict(part="train", n=1 << logM, layers=LAYERS, link_train_step_ms=float(np.median(step)) * 1e3,
             forward_backward_ms=float(np.median(ref)) * 1e3, ratio=float(np.median(step) / np.median(ref))))


def main():
    import torch

    from distributed_sddmm_b200 import driver as D
    print(json.dumps(dict(card=card())), flush=True)
    torch.cuda.set_device(0)
    D.world_init("self")
    out = lambda rec: print(json.dumps(rec), flush=True)  # noqa: E731
    parts = env("PARTS", "op,train").split(",")
    if "op" in parts:
        op_part(out)
    if "train" in parts:
        train_part(out)
    D.world_finalize()


if __name__ == "__main__":
    main()
