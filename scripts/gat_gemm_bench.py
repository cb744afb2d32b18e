#!/usr/bin/env python
"""CUDA-event time and fp64 throughput of the GAT backward GEMMs at the benchmark's layer shapes (rows = 2^LOGM):
hnh_dgemm_tn_f64 (weight gradient X^T dP: k = rows, m = input width, n = head width) and hnh_dgemm_nt_f64 (input
gradient dP W^T: m = rows, n = input width, k = head width), next to hnh_dgemm_f64 (the forward projection X W).
FLOPs = 2 m n k.  Prints one JSON line per (kernel, shape), after the card name and power limit.
Environment: LOGM (default 20), REPS (default 10)."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from distributed_sddmm_b200 import driver as D  # noqa: E402
from distributed_sddmm_b200 import lib  # noqa: E402

logM = int(os.environ.get("LOGM", "20"))
reps = int(os.environ.get("REPS", "10"))
rows = 1 << logM


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def timed(fn):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    L = lib()
    dev = torch.device("cuda:0")
    st = torch.cuda.current_stream().cuda_stream
    print(json.dumps({"device": torch.cuda.get_device_name(0), "power_limit": power_limit()}), flush=True)
    g = torch.Generator(device=dev).manual_seed(1)
    for width, head in ((1024, 256), (256, 256)):
        X = torch.rand((rows, width), generator=g, device=dev, dtype=torch.float64)
        dP = torch.rand((rows, head), generator=g, device=dev, dtype=torch.float64)
        W = torch.rand((width, head), generator=g, device=dev, dtype=torch.float64)
        dW = torch.empty((width, head), device=dev, dtype=torch.float64)
        dX = torch.empty((rows, width), device=dev, dtype=torch.float64)
        P = torch.empty((rows, head), device=dev, dtype=torch.float64)
        ws_bytes = L.hnh_dgemm_tn_workspace_bytes(width, head, rows)
        ws = torch.empty((max(ws_bytes, 8) // 8,), device=dev, dtype=torch.float64)
        runs = {
            "hnh_dgemm_tn_f64": lambda: D.check(L.hnh_dgemm_tn_f64(dW.data_ptr(), X.data_ptr(), dP.data_ptr(), width, head, rows,
                                                                   ws.data_ptr(), ws_bytes, st)),
            "hnh_dgemm_nt_f64": lambda: D.check(L.hnh_dgemm_nt_f64(dX.data_ptr(), dP.data_ptr(), W.data_ptr(), rows, width, head,
                                                                   0, st)),
            "hnh_dgemm_f64": lambda: D.check(L.hnh_dgemm_f64(P.data_ptr(), X.data_ptr(), W.data_ptr(), rows, head, width, st)),
        }
        for name, fn in runs.items():
            ms = timed(fn)
            flops = 2.0 * rows * width * head
            print(json.dumps({"kernel": name, "rows": rows, "width": width, "head": head, "ms": round(ms, 3),
                              "tflops": round(flops / ms / 1e9, 2)}), flush=True)
        del X, dP, W, dW, dX, P, ws
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
