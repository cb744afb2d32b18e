#!/usr/bin/env python
"""benchmark_algorithm (the reference's benchmark entry point, benchmark_dist.cpp:26-167) for the applications it
knows -- vanilla FusedMM, one ALS-CG round (run_cg(1): 2 x 10 batched CG iterations around fusedSpMM), the GAT
forward pass ("gat"), and one GAT training step ("gat_train": forward pass, then the backward pass for an all-ones
output gradient; the weights stay as "gat" leaves them) -- at the launched world size (torchrun).  One JSON record
per (application, algorithm) on rank 0.  Environment: LOGM, NPR, R, C, ALGS, APPS (e.g. APPS=gat,gat_train),
TRIALS, WARMUP."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from bench import SEED  # noqa: E402
from distributed_sddmm_b200 import driver as D  # noqa: E402

logM = int(os.environ.get("LOGM", "21"))
npr = int(os.environ.get("NPR", "32"))
R = int(os.environ.get("R", "128"))
c = int(os.environ.get("C", "1"))
algs = os.environ.get("ALGS", "15d_fusion2").split(",")
apps = os.environ.get("APPS", "vanilla,als").split(",")
trials = int(os.environ.get("TRIALS", "3"))
warmup = int(os.environ.get("WARMUP", "1"))

torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
rank, world = D.world_init()
S = D.SpmatLocal.load_er(logM, npr, SEED)
for app in apps:
    for alg in algs:
        try:
            rec = D.benchmark_algorithm(S, alg, R, c, fused=True, app=app, trials=trials, warmup=warmup)
        except RuntimeError as e:
            rec = {"error": str(e)[:300]}
        if rank == 0:
            keep = {k: rec.get(k) for k in ("elapsed", "overall_throughput", "num_trials", "warmup", "application_communication_time",
                                            "perf_stats", "error") if k in rec}
            # device memory in use after the run (cudaMemGetInfo): the library's caching allocator keeps what it
            # allocated, so this is close to the run's peak
            free_b, total_b = torch.cuda.mem_get_info()
            keep.update(app=app, alg=alg, logM=logM, nnz_per_row=npr, R=R, c=c, p=world,
                        ms_per_call=(rec["elapsed"] / rec["num_trials"] * 1e3) if "elapsed" in rec else None,
                        device_used_gib=round((total_b - free_b) / 2**30, 1))
            print(json.dumps(keep), flush=True)
del S
D.world_finalize()
