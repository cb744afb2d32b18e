#!/usr/bin/env python
"""CUDA-event time of the two GATv2 kernels on one GPU, each beside the existing kernel of the same shape on the same
CSR block and width: the scores (hnh_gatv2_scores_f64) beside the overwrite-form SDDMM (hnh_sddmm_f64 with
HNH_FLAG_BETA0), and the gradient gather (hnh_gatv2_grad_f64, with and without the da partials) beside the
accumulating SpMM (hnh_spmm_f64).  The block is the A order of an Erdos-Renyi 2^LOGM x 2^LOGM S with NPR draws per row
under ALG at p = 1 (15d_fusion1: 2^20 rows and 33 553 937 entries at the defaults), the dense operands one
2^LOGM x r matrix in both roles, at each r of WIDTHS.

Algorithmic bytes per call, from the shapes (int64 indices, fp64 values; a gathered row counted once per entry, as if
no cache held it):
    sddmm (overwrite)  nnz (8 col + 8 value + 8 r gathered) + rows (8 row start + 8 r row side)
    gatv2 scores       the SDDMM's + 8 r (a)
    spmm (accumulate)  nnz (8 col + 8 value + 8 r gathered) + rows (8 row start + 16 r output read and write)
    gatv2 grad         the SpMM's + rows 8 r (row side) + 8 r (a); with da, + CTAs 8 r (partials) read and written
They are set against the H100 SXM's 3.35 TB/s (a gathered row served from L2 can put a share above 1).  Prints the card
name and power limit, then one JSON line per kernel and width.  Environment: LOGM (20), NPR (32), WIDTHS (128,256),
ALG (15d_fusion1), REPS (20)."""
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from bench import SEED  # noqa: E402
from distributed_sddmm_b200 import driver as D  # noqa: E402
from distributed_sddmm_b200 import lib  # noqa: E402

logM = int(os.environ.get("LOGM", "20"))
npr = int(os.environ.get("NPR", "32"))
widths = [int(x) for x in os.environ.get("WIDTHS", "128,256").split(",")]
alg_name = os.environ.get("ALG", "15d_fusion1")
reps = int(os.environ.get("REPS", "20"))
HBM = 3.35e12
BETA0 = 4

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
# the CSR block that holds the A order (fusion 1 keeps it in ST's block, stored transposed: S-rows as stored rows)
blocks = [b for b in alg.blocks("ST" if alg_name == "15d_fusion1" else "S") if b is not None]
assert len(blocks) == 1, "one local block at p = 1"
blk = blocks[0]
rows, nnz = int(blk["rows"]), len(blk["col_idx"])
rs = torch.from_numpy(blk["rowStart"]).to(dev)
ci = torch.from_numpy(blk["col_idx"]).to(dev)
del blocks, blk, alg, S
st = torch.cuda.current_stream().cuda_stream
f64 = dict(dtype=torch.float64, device=dev)


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


def report(kernel, r, ms, nbytes, **extra):
    print(json.dumps(dict(kernel=kernel, logM=logM, nnz_per_row=npr, rows=rows, entries=nnz, r=r, ms_per_call=round(ms, 4),
                          min_bytes=nbytes, tb_per_s=round(nbytes / (ms * 1e-3) / 1e12, 3),
                          share_of_3_35_tb_s=round(nbytes / (ms * 1e-3) / HBM, 3), **extra)), flush=True)
    return ms


g = torch.Generator(device=dev).manual_seed(1)
values = torch.rand(nnz, generator=g, **f64)
out = torch.empty(nnz, **f64)
for r in widths:
    P = torch.rand((M, r), generator=g, **f64) * 2 - 1
    Q = torch.zeros((M, r), **f64)
    a = torch.rand(r, generator=g, **f64) * 2 - 1
    da = torch.zeros(r, **f64)
    ws_bytes = L.hnh_gatv2_grad_workspace_bytes(rows, r)
    ws = torch.empty(max(ws_bytes // 8, 1), **f64)
    per_entry, per_row = nnz * (16 + 8 * r), rows * 8
    sddmm = report("sddmm_overwrite", r, timed(lambda: D.check(L.hnh_sddmm_f64(
        rs.data_ptr(), ci.data_ptr(), out.data_ptr(), rows, nnz, P.data_ptr(), P.data_ptr(), r, BETA0, st))),
        per_entry + per_row + rows * 8 * r)
    scores = report("gatv2_scores", r, timed(lambda: D.check(L.hnh_gatv2_scores_f64(
        rs.data_ptr(), ci.data_ptr(), rows, nnz, P.data_ptr(), r, P.data_ptr(), r, a.data_ptr(), r, 0.2, out.data_ptr(), st))),
        per_entry + per_row + rows * 8 * r + 8 * r)
    spmm = report("spmm_accumulate", r, timed(lambda: D.check(L.hnh_spmm_f64(
        rs.data_ptr(), ci.data_ptr(), values.data_ptr(), rows, nnz, P.data_ptr(), Q.data_ptr(), r, 0, st))),
        per_entry + per_row + rows * 16 * r)
    grad_bytes = per_entry + per_row + rows * 24 * r + 8 * r
    grad = report("gatv2_grad", r, timed(lambda: D.check(L.hnh_gatv2_grad_f64(
        rs.data_ptr(), ci.data_ptr(), values.data_ptr(), rows, nnz, P.data_ptr(), r, P.data_ptr(), r, a.data_ptr(), r, 0.2,
        Q.data_ptr(), r, None, None, 0, st))), grad_bytes)
    grad_da = report("gatv2_grad_with_da", r, timed(lambda: D.check(L.hnh_gatv2_grad_f64(
        rs.data_ptr(), ci.data_ptr(), values.data_ptr(), rows, nnz, P.data_ptr(), r, P.data_ptr(), r, a.data_ptr(), r, 0.2,
        Q.data_ptr(), r, da.data_ptr(), ws.data_ptr(), ws_bytes, st))), grad_bytes + 2 * ws_bytes)
    print(json.dumps(dict(r=r, scores_over_sddmm=round(scores / sddmm, 3), grad_over_spmm=round(grad / spmm, 3),
                          grad_with_da_over_spmm=round(grad_da / spmm, 3))), flush=True)
    del P, Q, ws
D.world_finalize()
