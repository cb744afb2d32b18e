#!/usr/bin/env python
"""R-GCN with basis decomposition on one GPU: the basis-aggregation kernels against the accumulating SpMM and the
relational-aggregation kernel on the same block, the keyed reduction of the products into dcomp, and the basis model's
train step beside the model without bases.  Prints the card name and power limit first, then one JSON line per
measurement.

kernels (an Erdos-Renyi 2^LOGM x 2^LOGM block with NPR draws per row, relations uniform at random in [0, R), (B, f) in
BFS, REPS launches between CUDA events):
  - fwd: hnh_basis_aggregate_f64 adding into H (B f wide) with the mean's scale; grad: hnh_basis_aggregate_grad_f64 adding
    into dX with H as dH, the scale, and the per-entry products; spmm: hnh_spmm_f64 accumulating into Y on the same block
    and X; rel: hnh_relational_aggregate_f64 into A (R f wide) on the same block and X;
  - the share of 3.35 TB/s on each kernel's algorithmic bytes:
        fwd    nnz (16 + 8 f) + 8 (rows + 1) + 16 rows B f + 8 W   (col_idx and value, the gathered rows; rowStart; each
                                                                  row's B windows read and written once; the scale of
                                                                  each of the W distinct (stored row, relation) pairs)
        grad   nnz (24 + 8 B f + 8 B) + 8 (rows + 1) + 24 rows f   (col_idx, value and gathered scale, the B gathered dH
                                                                  windows and the B products of every entry; rowStart;
                                                                  X read and dX read and written)
        spmm   nnz (16 + 8 f) + 8 (rows + 1) + 16 rows f
        rel    nnz (16 + 8 f) + 8 (rows + 1) + 16 f W
    W is counted on the host from the tuples.
  - plan: the keyed reduction of the products into dcomp as basisAggregateBackward runs it: the relation keys, the
    edge-softmax plan over R + 1 keys (it synchronises) and B edge sums, timed on the host clock around a synchronise.
train (2^TRAIN_LOGM nodes, NPR draws per row, GraphSAGE's bench widths 256 -> 1024 -> 1024 -> 1536, 15d_fusion1 at
  p = 1, the mean): the median of TRIALS train_step calls of R-GCN with TRAIN_R relations and TRAIN_B bases, and of
  R-GCN without bases at PLAIN_R relations.  Both keep B f (or R f) doubles per row per layer: at 4 windows of 1024,
  2^18 x 4096 doubles (8.6 GB) per layer.  Without bases, TRAIN_R = 32 would keep 2^18 x 32768 doubles (68.7 GB) per
  layer and does not fit on one 80 GB card.

Environment: PARTS (kernels,plan,train), LOGM (20), NPR (32), R (32), BFS (4:128,8:128,30:16), REPS (20),
TRAIN_LOGM (18), TRAIN_R (32), TRAIN_B (4), PLAIN_R (4), TRIALS (3)."""
import ctypes as C
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


def fwd_bytes(nnz, rows, f, B, W):
    return nnz * (16 + 8 * f) + 8 * (rows + 1) + 16 * rows * B * f + 8 * W


def grad_bytes(nnz, rows, f, B):
    return nnz * (24 + 8 * B * f + 8 * B) + 8 * (rows + 1) + 24 * rows * f


def spmm_bytes(nnz, rows, f):
    return nnz * (16 + 8 * f) + 8 * (rows + 1) + 16 * rows * f


def rel_bytes(nnz, rows, f, W):
    return nnz * (16 + 8 * f) + 8 * (rows + 1) + 16 * f * W


def block(logM, npr, R):
    """The sorted ER block on the device: (n, nnz, rowStart, col, weights, relations, W)."""
    import numpy as np
    import torch

    from distributed_sddmm_b200 import driver as D
    S = D.SpmatLocal.load_er(logM, npr, 0xC0FFEE)
    rows_g, cols_g, vals_g = S.tuples()
    order = np.lexsort((cols_g, rows_g))
    n = 1 << logM
    rows_s = rows_g[order].astype(np.int64)
    rowStart = torch.from_numpy(np.searchsorted(rows_s, np.arange(n + 1)).astype(np.int64)).cuda()
    col = torch.from_numpy(cols_g[order].astype(np.int64)).cuda()
    vals = torch.from_numpy(vals_g[order]).cuda()
    rel_h = np.random.default_rng(5).integers(0, R, len(col))
    W = len(np.unique(rows_s * R + rel_h))
    counts = np.zeros((n, R))
    np.add.at(counts, (rows_s, rel_h), 1.0)
    scale = torch.from_numpy(np.divide(1.0, counts, out=np.zeros_like(counts), where=counts != 0)).cuda()
    return n, len(col), rowStart, col, vals, torch.from_numpy(rel_h.astype(np.float64)).cuda(), scale, W


def kernels_part(out, blk):
    import torch

    from distributed_sddmm_b200 import check, lib
    n, nnz, rowStart, col, vals, rel, scale, W = blk
    R, reps = int(env("R", "32")), int(env("REPS", "20"))
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

    for bf in env("BFS", "4:128,8:128,30:16").split(","):
        B, f = (int(x) for x in bf.split(":"))
        gen = torch.Generator(device="cuda").manual_seed(f + B)
        X = torch.randn((n, f), dtype=torch.float64, device="cuda", generator=gen)
        comp = torch.randn((R, B), dtype=torch.float64, device="cuda", generator=gen)
        H = torch.zeros((n, B * f), dtype=torch.float64, device="cuda")
        P = torch.zeros((B, nnz), dtype=torch.float64, device="cuda")
        Y, dX = torch.zeros_like(X), torch.zeros_like(X)
        fwd = lambda: L.hnh_basis_aggregate_f64(rowStart.data_ptr(), col.data_ptr(), rel.data_ptr(), n, nnz, X.data_ptr(), f, f,  # noqa: E731
                                                scale.data_ptr(), R, comp.data_ptr(), R, B, H.data_ptr(), B * f, st)
        grad = lambda: L.hnh_basis_aggregate_grad_f64(rowStart.data_ptr(), col.data_ptr(), rel.data_ptr(), n, nnz, H.data_ptr(),  # noqa: E731
                                                      B * f, scale.data_ptr(), R, comp.data_ptr(), R, B, X.data_ptr(), f, f,
                                                      dX.data_ptr(), f, P.data_ptr(), nnz, st)
        check(fwd(), "basis_aggregate")
        check(grad(), "basis_aggregate_grad")
        t_fwd, t_grad = kern(fwd), kern(grad)
        t_spmm = kern(lambda: L.hnh_spmm_f64(rowStart.data_ptr(), col.data_ptr(), vals.data_ptr(), n, nnz, X.data_ptr(), Y.data_ptr(),
                                             f, 0, st))
        del H, P
        A = torch.zeros((n, R * f), dtype=torch.float64, device="cuda")
        check(L.hnh_relational_aggregate_f64(rowStart.data_ptr(), col.data_ptr(), rel.data_ptr(), n, nnz, X.data_ptr(), f, f, R,
                                             A.data_ptr(), R * f, st), "relational_aggregate")
        t_rel = kern(lambda: L.hnh_relational_aggregate_f64(rowStart.data_ptr(), col.data_ptr(), rel.data_ptr(), n, nnz, X.data_ptr(),
                                                            f, f, R, A.data_ptr(), R * f, st))
        out(dict(part="kernels", R=R, B=B, f=f, n=n, nnz=nnz, windows=W, fwd_ms=t_fwd * 1e3, grad_ms=t_grad * 1e3,
                 spmm_ms=t_spmm * 1e3, rel_ms=t_rel * 1e3, fwd_over_spmm=t_fwd / t_spmm, grad_over_spmm=t_grad / t_spmm,
                 fwd_over_rel=t_fwd / t_rel, fwd_hbm_share=fwd_bytes(nnz, n, f, B, W) / t_fwd / HBM,
                 grad_hbm_share=grad_bytes(nnz, n, f, B) / t_grad / HBM, spmm_hbm_share=spmm_bytes(nnz, n, f) / t_spmm / HBM,
                 rel_hbm_share=rel_bytes(nnz, n, f, W) / t_rel / HBM))
        del X, A, Y, dX


def plan_part(out, blk):
    import torch

    from distributed_sddmm_b200 import check, lib
    n, nnz, rowStart, col, vals, rel, scale, W = blk
    R = int(env("R", "32"))
    st = torch.cuda.current_stream().cuda_stream
    L = lib()
    keys_n = R + 1
    i32 = dict(dtype=torch.int32, device="cuda")
    keys, perm = torch.empty(nnz, **i32), torch.empty(nnz, **i32)
    row_start, piece_first = torch.empty(keys_n + 1, **i32), torch.empty(keys_n + 1, **i32)
    piece_row = torch.empty(max(L.hnh_edge_softmax_piece_bound(nnz, keys_n), 1), **i32)
    for B in sorted({int(bf.split(":")[0]) for bf in env("BFS", "4:128,8:128,30:16").split(",")}):
        P = torch.randn((B, nnz), dtype=torch.float64, device="cuda")
        sums = torch.empty((B, keys_n), dtype=torch.float64, device="cuda")
        piece = torch.empty(max(len(piece_row), 1), dtype=torch.float64, device="cuda")
        pieces = C.c_int64()

        def run():
            check(L.hnh_relation_keys(keys.data_ptr(), rel.data_ptr(), nnz, R, st), "relation_keys")
            check(L.hnh_edge_softmax_plan(keys.data_ptr(), nnz, keys_n, perm.data_ptr(), row_start.data_ptr(), piece_first.data_ptr(),
                                          piece_row.data_ptr(), len(piece_row), C.byref(pieces), st), "edge_softmax_plan")
            for b in range(B):
                check(L.hnh_edge_sum_f64(P[b].data_ptr(), perm.data_ptr(), row_start.data_ptr(), piece_first.data_ptr(),
                                         piece_row.data_ptr(), keys_n, pieces.value, piece.data_ptr(), sums[b].data_ptr(), st),
                      "edge_sum")
        run()
        t = []
        for _ in range(5):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run()
            torch.cuda.synchronize()
            t.append(time.perf_counter() - t0)
        t.sort()
        out(dict(part="plan", R=R, B=B, nnz=nnz, pieces=pieces.value, plan_and_sums_ms=t[len(t) // 2] * 1e3))
        del P, sums, piece


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
    logM, npr, trials = int(env("TRAIN_LOGM", "18")), int(env("NPR", "32")), int(env("TRIALS", "3"))
    R, B, R_plain = int(env("TRAIN_R", "32")), int(env("TRAIN_B", "4")), int(env("PLAIN_R", "4"))
    S0 = D.SpmatLocal.load_er(logM, npr, 0xC0FFEE)
    rows, cols, _ = S0.tuples()
    del S0
    rng = np.random.default_rng(3)
    for model, nrel, nb in (("rgcn_basis_mean", R, B), ("rgcn_mean", R_plain, None)):
        S = D.SpmatLocal.from_tuples(1 << logM, 1 << logM, rows, cols, rng.integers(0, nrel, len(rows)).astype(np.float64))
        alg = D.Algorithm("15d_fusion1", S, LAYERS[0][0], 1)
        net = D.RGCN(alg, LAYERS, num_relations=nrel, aggr="mean", num_bases=nb)
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
        out(dict(part="train_step", model=model, relations=nrel, bases=nb, logM=logM, nnz_per_row=npr,
                 s_per_call=round(float(np.median(t)), 4)))
        del net, labels, opt, alg, S


def main():
    import torch

    from distributed_sddmm_b200 import driver as D
    print(json.dumps(dict(card=card())), flush=True)
    torch.cuda.set_device(0)
    D.world_init("self")
    out = lambda rec: print(json.dumps(rec), flush=True)  # noqa: E731
    parts = env("PARTS", "kernels,plan,train").split(",")
    if "kernels" in parts or "plan" in parts:
        blk = block(int(env("LOGM", "20")), int(env("NPR", "32")), int(env("R", "32")))
        if "kernels" in parts:
            kernels_part(out, blk)
        if "plan" in parts:
            plan_part(out, blk)
        del blk
        torch.cuda.empty_cache()  # the models allocate outside torch's cache
    if "train" in parts:
        train_part(out)
    D.world_finalize()


if __name__ == "__main__":
    main()
