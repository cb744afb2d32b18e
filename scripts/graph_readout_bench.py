"""Graph readout measurements (DESIGN.md §6): the pool forward (sum, max) and backward kernels at logM = 20 against the
one-row-per-graph baseline (hnh_spmm_f64 / hnh_max_aggregate_step_f64 on the same segment CSR), as a share of 3.35
TB/s on the minimal bytes, on three batches; and graph_train_step against train_step for GraphSAGE-mean on a
block-diagonal S at logM = 18.  One JSON line per measurement, with the card's name and power limit read in the same
run.  The batches are the shapes a readout meets: many small graphs (molecules), a few large ones, and one graph
holding half the nodes next to small ones, where one lane group per graph serialises on the big graph.

    python scripts/graph_readout_bench.py [--reps 30] [--steps 8]     (DESIGN §6 uses the defaults)
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from distributed_sddmm_b200 import driver as D  # noqa: E402
from distributed_sddmm_b200 import lib  # noqa: E402
from tests import graph_readout_oracle as gro  # noqa: E402

HBM = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (x.strip() for x in q.stdout.strip().splitlines()[0].split(","))
    return {"gpu": name, "power_limit": power}


def batches(n, rng):
    sizes = rng.integers(16, 49, n // 16)
    mol = np.repeat(np.arange(len(sizes)), sizes)[:n]
    few = np.repeat(np.arange(64), n // 64)
    half = n // 2
    small = rng.integers(16, 49, n // 16)
    skew = np.concatenate([np.zeros(half, np.int64), 1 + np.repeat(np.arange(len(small)), small)[:n - half]])
    return {"molecule": mol, "few_large": few, "skewed": skew}


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps * 1e-3


def check(rc):
    assert rc == 0, lib().hnh_last_error_string()


def pool_bench(info, reps):
    rng = np.random.default_rng(0)
    n = 1 << 20
    st = torch.cuda.current_stream().cuda_stream
    for name, batch in batches(n, rng).items():
        G = int(batch.max()) + 1
        seg_start, seg_rows, chunk_first, chunk_seg = (torch.from_numpy(a).cuda() for a in gro.plan(batch, G))
        vals = torch.ones(n, dtype=torch.float64, device="cuda")
        K = len(chunk_seg)
        for r in (64, 128, 256):
            H = torch.randn(n, r, dtype=torch.float64, device="cuda")
            P = torch.zeros(G, r, dtype=torch.float64, device="cuda")
            Cn = torch.zeros(G, r, dtype=torch.float64, device="cuda")
            nb = lib().hnh_segment_pool_workspace_bytes(K, r, 1)
            ws = torch.empty(max(nb // 8, 1), dtype=torch.float64, device="cuda")
            args = (seg_start.data_ptr(), seg_rows.data_ptr(), chunk_first.data_ptr(), chunk_seg.data_ptr(), G, K, H.data_ptr(), r, r,
                    P.data_ptr(), r)
            rg = torch.from_numpy(batch.astype(np.int32)).cuda()
            dH = torch.empty_like(H)
            runs = {
                "pool_sum": lambda: check(lib().hnh_segment_pool_f64(*args, None, r, ws.data_ptr(), nb, st)),
                "pool_max": lambda: check(lib().hnh_segment_pool_f64(*args, Cn.data_ptr(), r, ws.data_ptr(), nb, st)),
                "baseline_sum": lambda: check(lib().hnh_spmm_f64(seg_start.data_ptr(), seg_rows.data_ptr(), vals.data_ptr(), G, n,
                                                                 H.data_ptr(), P.data_ptr(), r, 0, st)),
                "baseline_max": lambda: check(lib().hnh_max_aggregate_step_f64(seg_start.data_ptr(), seg_rows.data_ptr(), G, n, H.data_ptr(),
                                                                               r, r, P.data_ptr(), r, Cn.data_ptr(), r, st)),
                "grad_sum": lambda: check(lib().hnh_segment_pool_grad_f64(rg.data_ptr(), n, G, P.data_ptr(), r, None, None, r, None, r,
                                                                          None, r, r, dH.data_ptr(), r, st)),
                "grad_max": lambda: check(lib().hnh_segment_pool_grad_f64(rg.data_ptr(), n, G, P.data_ptr(), r, None, H.data_ptr(), r,
                                                                          P.data_ptr(), r, Cn.data_ptr(), r, r, dH.data_ptr(), r, st)),
            }
            # minimal bytes: the pool reads H once and writes P (and C) once; the baselines also read the P (and C) they
            # add into (Y += ..., and the (max, count) merge); the backward reads dP (and H, P, C for max) and writes dH
            nbytes = {"pool_sum": (n + G) * r * 8, "pool_max": (n + 2 * G) * r * 8, "baseline_sum": (n + 2 * G) * r * 8,
                      "baseline_max": (n + 4 * G) * r * 8, "grad_sum": (n + G) * r * 8, "grad_max": (2 * n + 3 * G) * r * 8}
            for k, fn in runs.items():
                t = timed(fn, reps)
                print(json.dumps({**info, "measure": k, "batch": name, "graphs": G, "r": r, "logM": 20, "seconds": t,
                                  "hbm_share": nbytes[k] / t / HBM}), flush=True)


def step_bench(info, reps):
    rng = np.random.default_rng(1)
    logM, f, layers = 18, 64, [(64, 128), (128, 128), (128, 16)]
    n = 1 << logM
    sizes = rng.integers(16, 49, n // 16)
    batch = np.repeat(np.arange(len(sizes)), sizes)[:n]
    G = int(batch.max()) + 1
    # block-diagonal S: 8 random entries per row inside each graph
    starts = np.concatenate([[0], np.cumsum(np.bincount(batch))])[batch]
    lens = np.bincount(batch)[batch]
    rows = np.repeat(np.arange(n), 8)
    cols = starts.repeat(8) + rng.integers(0, 1 << 30, 8 * n) % lens.repeat(8)
    S = D.SpmatLocal.from_tuples(n, n, rows, cols, np.ones(len(rows)))
    alg = D.Algorithm("15d_fusion1", S, f, 1)
    net = D.GraphSAGE(alg, layers, aggr="mean")
    for l, (fi, r) in enumerate(layers):
        for k, shape in (("neigh", (fi, r)), ("neigh_bias", (r,)), ("root", (fi, r))):
            net.set_param(l, k, rng.uniform(-1, 1, shape) / np.sqrt(fi))
    net.set_input(rng.uniform(-1, 1, net.buffer_shape(0)))
    rows_out = net.buffer_shape(len(layers))[0]
    node_labels = D.NodeLabels(net, np.where(np.arange(rows_out) < n, rng.integers(0, 16, rows_out), -1), 16)
    b = np.full(rows_out, -1, np.int64)
    b[:n] = batch
    ro = D.GraphReadout(net, b, G, pool="mean", num_classes=16)
    graph_labels = D.GraphLabels(ro, rng.integers(0, 16, G), 16)
    o1, o2 = D.AdamW(lr=1e-3), D.AdamW(lr=1e-3)
    steps = {"node_step": lambda: net.train_step(node_labels, o1), "graph_step": lambda: net.graph_train_step(ro, graph_labels, o2)}
    for fn in steps.values():
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in steps}
    for _ in range(reps):  # alternated, so both see the same machine
        for k, fn in steps.items():
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[k].append(time.perf_counter() - t0)
    med = {k: float(np.median(v)) for k, v in times.items()}
    for k, v in med.items():
        print(json.dumps({**info, "measure": k, "model": "GraphSAGE-mean", "layers": layers, "logM": logM, "graphs": G,
                          "seconds_median": v, "ratio_to_node_step": v / med["node_step"]}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--steps", type=int, default=8)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the measurements need a GPU"
    info = card()
    D.world_init("self")
    pool_bench(info, a.reps)
    step_bench(info, a.steps)
    D.world_finalize()


if __name__ == "__main__":
    main()
