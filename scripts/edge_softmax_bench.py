#!/usr/bin/env python
"""CUDA-event time of Algorithm.edge_softmax and edge_softmax_backward on one rank at the GAT benchmark's size
(Erdos-Renyi 2^LOGM x 2^LOGM, NPR draws per row), per value order, over REPS calls after a warm-up call (which also
builds the order's row grouping; its wall time is reported as plan_s).  Bytes per call are what the kernels must
move at least, from the sizes: forward 32 per entry (perm 4 + gathered score 8 in the row pass; score 8 + key 4 +
alpha 8 in the apply pass) and backward 48 per entry (perm 4 + alpha 8 + grad 8; alpha 8 + grad 8 + key 4 + out 8),
plus 40 per row for the row statistics; they are set against the H100 SXM's 3.35 TB/s.  Prints the card name and
power limit, then one JSON line per (order, direction).  Environment: LOGM (default 20), NPR (32), ALG (15d_fusion1),
REPS (10)."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import SEED  # noqa: E402
from distributed_sddmm_b200 import driver as D  # noqa: E402

logM = int(os.environ.get("LOGM", "20"))
npr = int(os.environ.get("NPR", "32"))
alg_name = os.environ.get("ALG", "15d_fusion1")
reps = int(os.environ.get("REPS", "10"))
HBM = 3.35e12

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True, timeout=30).stdout.strip()
print(json.dumps({"card": card}), flush=True)
torch.cuda.set_device(0)
D.world_init("self")
S = D.SpmatLocal.load_er(logM, npr, SEED)
alg = D.Algorithm(alg_name, S, 32, 1)
M = alg.dims.M
for mode in ("A", "B"):
    like = alg.like_S_values if mode == "A" else alg.like_ST_values
    x, g = like(0.0), like(0.0)
    n = len(x)
    rng = np.random.default_rng(1)
    x.from_host(rng.uniform(-50, 50, n))
    g.from_host(rng.uniform(-1, 1, n))
    D.check(D.lib().hnhd_device_synchronize())
    t0 = time.perf_counter()
    alg.edge_softmax(x, mode)  # builds the plan of this order
    D.check(D.lib().hnhd_device_synchronize())
    plan_s = time.perf_counter() - t0
    for direction, call, per_entry in (("forward", lambda: alg.edge_softmax(x, mode), 32),
                                       ("backward", lambda: alg.edge_softmax_backward(x, g, mode), 48)):
        call()
        D.timer_start()
        for _ in range(reps):
            call()
        ms = D.timer_stop() / reps
        nbytes = per_entry * n + 40 * M
        print(json.dumps(dict(alg=alg_name, order=mode, direction=direction, logM=logM, nnz_per_row=npr, entries=n,
                              ms_per_call=round(ms, 4), plan_s=round(plan_s, 3), min_bytes=nbytes,
                              tb_per_s=round(nbytes / (ms * 1e-3) / 1e12, 3),
                              share_of_3_35_tb_s=round(nbytes / (ms * 1e-3) / HBM, 3))), flush=True)
del alg, S
D.world_finalize()
