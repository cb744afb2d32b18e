#!/usr/bin/env python
"""Step time of the graph transformer against GAT with softmax attention, and the bytes/s of the gate and LayerNorm
kernels, on one GPU.

Apps (benchmark_algorithm, GAT's layer shapes (256, 256, 4), (1024, 256, 4), (1024, 256, 6), no edge features, no
gate, zero parameters): graph_transformer_train, graph_transformer (forward only) and gat_softmax_train, each on an
Erdos-Renyi 2^LOGM x 2^LOGM S with NPR draws per row under ALG at p = 1, each in a process of its own, WARMUP untimed and
TRIALS timed calls; one JSON line per app with the seconds per call and the device memory the process holds at the end
(the library's allocator caches every block it frees, so this is its high-water mark unless it had to give the cache
back).  The graph transformer keeps M and L of every layer and, in the backward of the widest layer, Q, K, V, dQ, dK, dV
and dM beside them: 2^20 rows do not fit in 80 GB; 2^18 do.

Gate kernels (hnh_gt_gate_f64 with the gate and the ReLU; hnh_gt_gate_backward_f64 with both), on 2^GATE_LOGM rows of
width GATE_R, REPS launches each.  Algorithmic bytes: forward 24 r per row (M, R read, Y written), backward 48 r per
row (G, Y, M, R read, dM, dR written); set against the H100 SXM's 3.35 TB/s.  Prints the card name and power limit
first.

The apps graph_transformer_block and graph_transformer_block_train (the same layers as transformer blocks with
ffn_ratio = 2) may be named in APPS.  PARTS=norm times the LayerNorm kernels on 2^GATE_LOGM rows of width GATE_R:
hnh_layer_norm_f64 without and with the residual (minimal bytes 16 r and 24 r per row: X (and Res) read, Y written;
the 16 bytes of (mean, rstd) per row are not counted) and hnh_layer_norm_backward_f64 overwriting and adding to dX
(24 r and 32 r per row: G and X read, dX written (and read)).

Environment: LOGM (18), NPR (32), ALG (15d_fusion1), TRIALS (3), WARMUP (1), GATE_LOGM (20), GATE_R (1024), REPS (20),
APPS (graph_transformer_train,graph_transformer,gat_softmax_train), PARTS (apps,gate)."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM = 3.35e12


def env(name, default):
    return os.environ.get(name, default)


def run_app(app):
    import torch

    from bench import SEED
    from distributed_sddmm_b200 import driver as D
    torch.cuda.set_device(0)
    D.world_init("self")
    logM, npr = int(env("LOGM", "18")), int(env("NPR", "32"))
    S = D.SpmatLocal.load_er(logM, npr, SEED)
    rec = D.benchmark_algorithm(S, env("ALG", "15d_fusion1"), R=256, c=1, fused=True, app=app,
                                trials=int(env("TRIALS", "3")), warmup=int(env("WARMUP", "1")))
    free, total = torch.cuda.mem_get_info()
    print(json.dumps(dict(app=app, logM=logM, nnz_per_row=npr, alg=env("ALG", "15d_fusion1"),
                          s_per_call=round(rec["elapsed"] / rec["num_trials"], 4), trials=rec["num_trials"],
                          device_gb_held=round((total - free) / 1e9, 2))), flush=True)
    D.world_finalize()


def gate():
    import numpy as np
    import torch

    from distributed_sddmm_b200 import check, lib
    L = lib()
    n, r, reps = 1 << int(env("GATE_LOGM", "20")), int(env("GATE_R", "1024")), int(env("REPS", "20"))
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(7)
    M, R, G = (torch.rand((n, r), generator=g, device=dev, dtype=torch.float64) - 0.5 for _ in range(3))
    w = torch.rand(3 * r, generator=g, device=dev, dtype=torch.float64) - 0.5
    Y, dM, dR = (torch.empty((n, r), device=dev, dtype=torch.float64) for _ in range(3))
    dw = torch.empty(3 * r, device=dev, dtype=torch.float64)
    ws_bytes = L.hnh_gt_gate_backward_workspace_bytes(n, r)
    ws = torch.empty(max(ws_bytes, 8) // 8, device=dev, dtype=torch.float64)
    st = torch.cuda.current_stream().cuda_stream

    def fwd():
        check(L.hnh_gt_gate_f64(Y.data_ptr(), M.data_ptr(), R.data_ptr(), w.data_ptr(), n, r, 1, st), "gate")

    def bwd():
        check(L.hnh_gt_gate_backward_f64(dM.data_ptr(), dR.data_ptr(), dw.data_ptr(), G.data_ptr(), Y.data_ptr(), M.data_ptr(),
                                         R.data_ptr(), w.data_ptr(), n, r, 1, ws.data_ptr(), ws_bytes, st), "gate_backward")

    for name, call, nbytes in (("gate", fwd, 24 * n * r), ("gate_backward", bwd, 48 * n * r)):
        time_kernel(name, call, n, r, nbytes, reps)
    assert np.isfinite(dw.cpu().numpy()).all()


def time_kernel(name, call, n, r, nbytes, reps):
    """One warm-up call, then `reps` calls between CUDA events; prints one JSON line."""
    import torch
    call()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        call()
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / reps
    print(json.dumps(dict(kernel=name, rows=n, r=r, ms_per_call=round(ms, 4), min_bytes=nbytes,
                          tb_per_s=round(nbytes / (ms * 1e-3) / 1e12, 3),
                          share_of_3_35_tb_s=round(nbytes / (ms * 1e-3) / HBM, 3))), flush=True)


def norm():
    import numpy as np
    import torch

    from distributed_sddmm_b200 import check, lib
    L = lib()
    n, r, reps = 1 << int(env("GATE_LOGM", "20")), int(env("GATE_R", "1024")), int(env("REPS", "20"))
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(11)
    X, Res, G = (torch.rand((n, r), generator=g, device=dev, dtype=torch.float64) - 0.5 for _ in range(3))
    gamma, beta = (torch.rand(r, generator=g, device=dev, dtype=torch.float64) + 0.5 for _ in range(2))
    Y, dX = (torch.empty((n, r), device=dev, dtype=torch.float64) for _ in range(2))
    stats = torch.empty((n, 2), device=dev, dtype=torch.float64)
    dgamma, dbeta = (torch.empty(r, device=dev, dtype=torch.float64) for _ in range(2))
    ws_bytes = L.hnh_layer_norm_backward_workspace_bytes(n, r)
    ws = torch.empty(max(ws_bytes, 8) // 8, device=dev, dtype=torch.float64)
    st = torch.cuda.current_stream().cuda_stream

    def fwd(res):
        return lambda: check(L.hnh_layer_norm_f64(Y.data_ptr(), stats.data_ptr(), X.data_ptr(), res, gamma.data_ptr(),
                                                  beta.data_ptr(), n, r, 1e-5, st), "layer_norm")

    def bwd(acc):
        return lambda: check(L.hnh_layer_norm_backward_f64(dX.data_ptr(), dgamma.data_ptr(), dbeta.data_ptr(), G.data_ptr(),
                                                           X.data_ptr(), None, stats.data_ptr(), gamma.data_ptr(), n, r, acc,
                                                           ws.data_ptr(), ws_bytes, st), "layer_norm_backward")

    time_kernel("layer_norm", fwd(None), n, r, 16 * n * r, reps)
    time_kernel("layer_norm_residual", fwd(Res.data_ptr()), n, r, 24 * n * r, reps)
    fwd(None)()  # the backward's statistics: those of X alone
    dX.zero_()
    time_kernel("layer_norm_backward", bwd(0), n, r, 24 * n * r, reps)
    time_kernel("layer_norm_backward_add", bwd(1), n, r, 32 * n * r, reps)
    assert np.isfinite(dgamma.cpu().numpy()).all() and np.isfinite(dX.cpu().numpy()).all()


def main():
    if len(sys.argv) > 2 and sys.argv[1] == "--app":
        return run_app(sys.argv[2])
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True, timeout=30).stdout.strip()
    print(json.dumps({"card": card}), flush=True)
    parts = env("PARTS", "apps,gate").split(",")
    if "apps" in parts:
        for app in env("APPS", "graph_transformer_train,graph_transformer,gat_softmax_train").split(","):
            subprocess.run([sys.executable, os.path.abspath(__file__), "--app", app], check=True)
    if "gate" in parts:
        gate()
    if "norm" in parts:
        norm()


if __name__ == "__main__":
    main()
