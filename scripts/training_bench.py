#!/usr/bin/env python
"""Training on one GPU: the device train step against the forward + backward it wraps and against the host loop it
replaces, and the bytes/s of the cross-entropy and AdamW kernels.  Prints the card name and power limit first.

fit (one process per model, GAT's layer shapes (256, 256, 4), (1024, 256, 4), (1024, 256, 6), so C = 1536, on an
Erdos-Renyi 2^LOGM x 2^LOGM S with NPR draws per row under 15d_fusion1 at p = 1; seeded small random parameters and
input, every node labelled; models graph_transformer (ffn_ratio 0), graph_transformer_block (ffn_ratio 2) and
gat_softmax):
  - train_step: net.train_step(labels, AdamW()), WARMUP untimed and TRIALS timed calls (each ends in a synchronise);
  - app: the benchmark app <model>_train (forward + backward from a gradient of ones), TRIALS timed calls;
  - host_loop: forward, download the output, torch's CPU cross-entropy gradient, upload it, backward, then read every
    gradient, torch's CPU AdamW(foreach=False) on every parameter and write every parameter back; HOST_TRIALS calls.
kernels: hnh_cross_entropy_f64 on 2^CE_LOGM rows at C in CE_C (minimal bytes 16 C + 4 per row: logits read, dlogits
written, the label read) and hnh_adamw_f64 on 2^ADAMW_LOGN parameters (56 bytes each: p, g, m, v read, p, m, v written),
REPS launches between CUDA events, against the H100 SXM's 3.35 TB/s.

Environment: PARTS (fit,kernels), MODELS (graph_transformer,graph_transformer_block,gat_softmax), LOGM (18), NPR (32),
TRIALS (3), WARMUP (1), HOST_TRIALS (1), CE_LOGM (20), CE_C (40,256,1536), ADAMW_LOGN (24), REPS (20)."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM = 3.35e12
LAYERS = [(256, 256, 4), (1024, 256, 4), (1024, 256, 6)]


def env(name, default):
    return os.environ.get(name, default)


def fit(model):
    import numpy as np
    import torch
    import torch.nn.functional as F

    from bench import SEED
    from distributed_sddmm_b200 import driver as D
    torch.cuda.set_device(0)
    D.world_init("self")
    logM, npr, trials = int(env("LOGM", "18")), int(env("NPR", "32")), int(env("TRIALS", "3"))
    S = D.SpmatLocal.load_er(logM, npr, SEED)
    alg = D.Algorithm("15d_fusion1", S, LAYERS[0][0], 1)
    rng = np.random.default_rng(5)
    if model == "gat_softmax":
        net = D.GAT(alg, LAYERS, attention="softmax")
        shapes = {(l, h): net.weight_shape(l, h) for l, (_, _, H) in enumerate(LAYERS) for h in range(H)}
        for (l, h), s in shapes.items():
            net.set_weight(l, h, rng.uniform(-1, 1, s) / np.sqrt(s[0]))
    else:
        net = D.GraphTransformer(alg, LAYERS, ffn_ratio=2 if model == "graph_transformer_block" else 0)
        for l in range(len(LAYERS)):
            for name in net.param_names():
                s = net.param_shape(l, name)
                if name not in ("norm1", "norm2"):
                    net.set_param(l, name, rng.uniform(-1, 1, s) * (0.05 if len(s) == 1 else 1 / np.sqrt(s[0])))
    net.set_input(rng.uniform(-1, 1, net.buffer_shape(0)))
    last = len(LAYERS)
    n, C = net.buffer_shape(last)
    lab = rng.integers(0, C, n)
    lab[1 << logM:] = -1
    labels, opt = D.NodeLabels(net, lab, C), D.AdamW()
    for _ in range(int(env("WARMUP", "1"))):
        net.train_step(labels, opt)
    t0 = time.perf_counter()
    for _ in range(trials):
        r = net.train_step(labels, opt)
    step = (time.perf_counter() - t0) / trials
    print(json.dumps(dict(model=model, part="train_step", logM=logM, nnz_per_row=npr, s_per_call=round(step, 4), loss=r.loss)),
          flush=True)

    # the host loop the train step replaces
    if model == "gat_softmax":
        names = [(l, h) for l, (_, _, H) in enumerate(LAYERS) for h in range(H)]
        get, grad, put = (lambda k: net.weight(*k)), (lambda k: net.weight_grad(*k)), (lambda k, v: net.set_weight(*k, v))
    else:
        names = [(l, name) for l in range(len(LAYERS)) for name in net.param_names()]
        get, grad, put = (lambda k: net.param(*k)), (lambda k: net.param_grad(*k)), (lambda k, v: net.set_param(*k, v))
    tp = {k: torch.from_numpy(get(k)) for k in names}
    host_opt = torch.optim.AdamW(list(tp.values()), foreach=False)
    labt = torch.from_numpy(np.where(lab < 0, -1, lab))
    host_trials = int(env("HOST_TRIALS", "1"))
    t0 = time.perf_counter()
    for _ in range(host_trials):
        net.forward()
        logits = torch.from_numpy(net.buffer(last)).requires_grad_()
        F.cross_entropy(logits, labt, ignore_index=-1).backward()
        net.backward(logits.grad.numpy())
        for k, t in tp.items():
            t.grad = torch.from_numpy(grad(k))
        host_opt.step()
        for k, t in tp.items():
            put(k, t.numpy())
    host = (time.perf_counter() - t0) / host_trials
    print(json.dumps(dict(model=model, part="host_loop", logM=logM, s_per_call=round(host, 4))), flush=True)
    del net, labels, opt
    rec = D.benchmark_algorithm(S, "15d_fusion1", R=256, c=1, fused=True, app=model + "_train", trials=trials, warmup=1)
    app = rec["elapsed"] / rec["num_trials"]
    print(json.dumps(dict(model=model, part="app", app=model + "_train", s_per_call=round(app, 4),
                          train_step_over_app=round(step / app, 4), host_loop_over_train_step=round(host / step, 3))), flush=True)
    D.world_finalize()


def time_kernel(name, call, nbytes, reps, **info):
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
    print(json.dumps(dict(kernel=name, **info, ms_per_call=round(ms, 4), min_bytes=nbytes,
                          tb_per_s=round(nbytes / (ms * 1e-3) / 1e12, 3),
                          share_of_3_35_tb_s=round(nbytes / (ms * 1e-3) / HBM, 3))), flush=True)


def kernels():
    import torch

    from distributed_sddmm_b200 import check, lib
    L = lib()
    dev = torch.device("cuda:0")
    reps = int(env("REPS", "20"))
    st = torch.cuda.current_stream().cuda_stream
    g = torch.Generator(device=dev).manual_seed(3)
    n = 1 << int(env("CE_LOGM", "20"))
    sums = torch.empty(2, device=dev, dtype=torch.float64)
    ws_bytes = L.hnh_cross_entropy_workspace_bytes(n)
    ws = torch.empty(ws_bytes // 8 + 1, device=dev, dtype=torch.float64)
    for C in (int(c) for c in env("CE_C", "40,256,1536").split(",")):
        x = torch.randn((n, C), generator=g, device=dev, dtype=torch.float64) * 3
        d = torch.empty_like(x)
        lab = torch.randint(-1, C, (n,), generator=g, device=dev, dtype=torch.int32)
        call = lambda: check(L.hnh_cross_entropy_f64(d.data_ptr(), sums.data_ptr(), x.data_ptr(), lab.data_ptr(), n, C, C,  # noqa: E731
                                                     1.0 / n, ws.data_ptr(), ws_bytes, st), "cross_entropy")
        time_kernel("cross_entropy", call, (16 * C + 4) * n, reps, rows=n, C=C)
        del x, d
    m = 1 << int(env("ADAMW_LOGN", "24"))
    P, G, M, V = (torch.randn(m, generator=g, device=dev, dtype=torch.float64) for _ in range(4))
    V.abs_()
    call = lambda: check(L.hnh_adamw_f64(P.data_ptr(), M.data_ptr(), V.data_ptr(), G.data_ptr(), m, 1e-3, 0.9, 0.999, 1e-8,  # noqa: E731
                                         1e-2, 0.5, 0.01, None, st), "adamw")
    time_kernel("adamw", call, 56 * m, reps, params=m)


def main():
    if len(sys.argv) > 2 and sys.argv[1] == "--fit":
        return fit(sys.argv[2])
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True, timeout=30).stdout.strip()
    print(json.dumps({"card": card}), flush=True)
    parts = env("PARTS", "fit,kernels").split(",")
    if "fit" in parts:
        for model in env("MODELS", "graph_transformer,graph_transformer_block,gat_softmax").split(","):
            subprocess.run([sys.executable, os.path.abspath(__file__), "--fit", model], check=True)
    if "kernels" in parts:
        kernels()


if __name__ == "__main__":
    main()
