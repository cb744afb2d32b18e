#!/usr/bin/env python
"""CUDA-event time of the additive-attention kernels on one GPU at the GAT benchmark's size: the node-scalar pair
s = P a1, t = P a2 (hnh_gat_node_scalars_f64) on a 2^LOGM x D projection, the edge scores LeakyReLU(s_u + t_v) and
their derivative (hnh_gat_edge_scores_f64), and the row and column sums of an A-order vector (hnh_edge_sum_f64, one
launch pair per grouping) on the A order of an Erdos-Renyi 2^LOGM x 2^LOGM S with NPR draws per row (about 2^25
entries at the defaults).  The keys and groupings are the library's own: read back through Algorithm.additive_scores
of index node vectors, grouped with hnh_edge_softmax_plan.  Bytes per call are what each kernel must move at least,
from the sizes: node scalars 8 n d + 16 n + 16 d; edge scores 16 per entry (two int32 keys, the output) + 16 per
node (s and t); a sum 12 per entry (perm 4, the value 8) + 12 per row or column (row start, pieces, output); they
are set against the H100 SXM's 3.35 TB/s.  Prints the card name and power limit, then one JSON line per kernel.
Environment: LOGM (default 20), NPR (32), D (256), ALG (15d_fusion1), REPS (20)."""
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import SEED  # noqa: E402
from distributed_sddmm_b200 import driver as D  # noqa: E402
from distributed_sddmm_b200 import lib  # noqa: E402

logM = int(os.environ.get("LOGM", "20"))
npr = int(os.environ.get("NPR", "32"))
d = int(os.environ.get("D", "256"))
alg_name = os.environ.get("ALG", "15d_fusion1")
reps = int(os.environ.get("REPS", "20"))
HBM = 3.35e12

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True, timeout=30).stdout.strip()
print(json.dumps({"card": card}), flush=True)
torch.cuda.set_device(0)
dev = torch.device("cuda:0")
D.world_init("self")
L = lib()
S = D.SpmatLocal.load_er(logM, npr, SEED)
alg = D.Algorithm(alg_name, S, 32, 1)
M = int(alg.dims.M)


def vec(n):
    h = C.c_void_p()
    D.check(L.hnhd_vec_create(n, 0.0, C.byref(h)))
    return D.Vec(h)


# the A order's row and column keys, as the library computes them
zero, index = vec(M), vec(M)
index.from_host(np.arange(M, dtype=np.float64))
out = alg.like_S_values(0.0)
keys = []
for s_vec, t_vec in ((index, zero), (zero, index)):
    alg.additive_scores(s_vec, t_vec, out, "A")
    keys.append(torch.from_numpy(np.rint(out.to_host()).astype(np.int32)).to(dev))
del out, zero, index
n = int(keys[0].numel())
st = torch.cuda.current_stream().cuda_stream
f64 = dict(dtype=torch.float64, device=dev)
I32 = dict(dtype=torch.int32, device=dev)


def timed(call):
    call()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        call()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / reps


def report(kernel, ms, nbytes, **extra):
    print(json.dumps(dict(kernel=kernel, logM=logM, nnz_per_row=npr, entries=n, d=d, ms_per_call=round(ms, 4), min_bytes=nbytes,
                          tb_per_s=round(nbytes / (ms * 1e-3) / 1e12, 3),
                          share_of_3_35_tb_s=round(nbytes / (ms * 1e-3) / HBM, 3), **extra)), flush=True)


# 1. node scalars
g = torch.Generator(device=dev).manual_seed(1)
P = torch.rand((M, d), generator=g, **f64) * 2 - 1
a = torch.rand((2, d), generator=g, **f64) * 2 - 1
s, t = torch.empty(M, **f64), torch.empty(M, **f64)
ms = timed(lambda: D.check(L.hnh_gat_node_scalars_f64(s.data_ptr(), t.data_ptr(), P.data_ptr(), a[0].data_ptr(), a[1].data_ptr(), M, d, st)))
report("node_scalars", ms, 8 * M * d + 16 * M + 16 * d)
del P

# 2. edge scores and their derivative
x = torch.empty(n, **f64)
for derivative in (0, 1):
    ms = timed(lambda: D.check(L.hnh_gat_edge_scores_f64(x.data_ptr(), s.data_ptr(), t.data_ptr(), keys[0].data_ptr(), keys[1].data_ptr(),
                                                         n, 0.2, derivative, st)))
    report("edge_scores", ms, 16 * n + 16 * M, derivative=derivative)

# 4. row and column sums of an A-order vector
for which, k in (("rows", keys[0]), ("columns", keys[1])):
    cap = L.hnh_edge_softmax_piece_bound(n, M)
    perm, rs, pf, pr = torch.empty(n, **I32), torch.empty(M + 1, **I32), torch.empty(M + 1, **I32), torch.empty(max(cap, 1), **I32)
    npieces = C.c_int64(-1)
    D.check(L.hnh_edge_softmax_plan(k.data_ptr(), n, M, perm.data_ptr(), rs.data_ptr(), pf.data_ptr(), pr.data_ptr(), cap,
                                    C.byref(npieces), st))
    ps, sums = torch.empty(max(npieces.value, 1), **f64), torch.empty(M, **f64)
    ms = timed(lambda: D.check(L.hnh_edge_sum_f64(x.data_ptr(), perm.data_ptr(), rs.data_ptr(), pf.data_ptr(), pr.data_ptr(), M,
                                                  npieces.value, ps.data_ptr(), sums.data_ptr(), st)))
    report("edge_sum", ms, 12 * n + 12 * M, grouping=which, pieces=npieces.value)
    del perm, rs, pf, pr, ps, sums
del alg, S
D.world_finalize()
