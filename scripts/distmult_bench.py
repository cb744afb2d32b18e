#!/usr/bin/env python
"""Relation-aware link prediction on one GPU: the DistMult decoder's kernels, the op against the torch composition, and
an R-GCN relational link train step against its dot-product link train step.  Prints the card name and power limit
first, then one JSON line per measurement.

kernels (an Erdos-Renyi 2^LOGM x 2^LOGM target matrix T with NPR draws per row, r = R_WIDTH, relations drawn uniformly
from [0, R) for R in RELS, under 15d_fusion1 at p = 1; H random, H_A = H_B = H):
  - kernel_fwd: hnh_distmult_bce_f64 with dX, stats, scores and g (the A-order pass); kernel_grad: hnh_distmult_bce_grad_f64
    (the B-order pass; the same block here); kernel_link: hnh_link_bce_f64 with dX and stats on the same block; each
    REPS launches between CUDA events.  Share of 3.35 TB/s on each pass's minimal bytes: the row side read once and its
    gradient read and written (3 n r 8), every gathered row (nnz r 8), col_idx and the values (nnz 16), rowStart (n 8),
    the stats (n 16 read and written) and for the forward the scores and g (nnz 16); D (R r 8) is read once;
  - dD_pass: Algorithm.distmult_loss with dH and dD minus the same call without dD (both synchronised): the relation
    plan, which this call builds afresh (RelationalLinkTargets builds it once), and the relation-gradient pass
    (hnh_distmult_relation_grad_f64: two gathered rows and g per entry, nnz (2 r 8 + 24) bytes); its ratio to kernel_grad;
  - op: Algorithm.distmult_loss with dH and dD against the torch composition (index_select, mul, sum,
    binary_cross_entropy_with_logits, autograd) on the same data, forward plus backward, both ending in a synchronise.
train (2^TRAIN_LOGM nodes, S Erdos-Renyi with NPR_S draws per row and R_TRAIN hashed relations, T_pos and T_neg of
  NPR_T draws per row, R-GCN with layers TRAIN_LAYERS): the median of TRIALS relational_link_train_step calls against
  link_train_step on one target matrix holding the same pairs.

Environment: PARTS (kernels,op,train), LOGM (20), NPR (32), R_WIDTH (128), RELS (1,16,237), REPS (10), TRIALS (5),
TRAIN_LOGM (16), NPR_S (16), NPR_T (8), R_TRAIN (8)."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM = 3.35e12
TRAIN_LAYERS = [(64, 64), (64, 64)]


def env(name, default):
    return os.environ.get(name, default)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timed(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps


def event_time(fn, reps):
    import torch
    fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 1e3 / reps


def kernels_and_op(out, parts):
    import numpy as np
    import torch
    import torch.nn.functional as F

    from distributed_sddmm_b200 import check, lib
    from distributed_sddmm_b200 import driver as D
    logM, npr, reps, r = int(env("LOGM", "20")), int(env("NPR", "32")), int(env("REPS", "10")), int(env("R_WIDTH", "128"))
    n = 1 << logM
    T1 = D.SpmatLocal.load_er(logM, npr, 0xC0FFEE)
    rows_g, cols_g, _ = T1.tuples()
    order = np.lexsort((cols_g, rows_g))
    rows_g, cols_g = rows_g[order].astype(np.int64), cols_g[order].astype(np.int64)
    del T1, order
    nnz = len(cols_g)
    rowStart = torch.from_numpy(np.searchsorted(rows_g, np.arange(n + 1)).astype(np.int64)).cuda()
    col = torch.from_numpy(cols_g).cuda()
    st = torch.cuda.current_stream().cuda_stream
    rng = np.random.default_rng(1)
    X = torch.from_numpy(rng.standard_normal((n, r)) / np.sqrt(r)).cuda()
    dX = torch.zeros_like(X)
    stats = torch.zeros((n, 2), dtype=torch.float64, device="cuda")
    scores = torch.zeros(nnz, dtype=torch.float64, device="cuda")
    g = torch.zeros(nnz, dtype=torch.float64, device="cuda")
    ones = torch.ones(nnz, dtype=torch.float64, device="cuda")
    L = lib()
    inv = 1.0 / nnz
    base = 3 * n * r * 8 + nnz * r * 8 + nnz * 16 + n * 8 + n * 32
    link = event_time(lambda: check(L.hnh_link_bce_f64(rowStart.data_ptr(), col.data_ptr(), ones.data_ptr(), n, nnz, X.data_ptr(), r,
                                                       X.data_ptr(), r, r, inv, dX.data_ptr(), r, stats.data_ptr(), 2, None, st),
                                    "link_bce"), reps)
    for R in [int(x) for x in env("RELS", "1,16,237").split(",")]:
        rels_np = rng.integers(0, R, nnz).astype(np.float64)
        rels = torch.from_numpy(rels_np).cuda()
        Dt = torch.from_numpy(rng.uniform(0.5, 1.5, (R, r))).cuda()
        rec = dict(part="kernels", logM=logM, npr=npr, nnz=nnz, r=r, R=R)
        fwd = grad = None
        if "kernels" in parts:
            fwd = event_time(lambda: check(L.hnh_distmult_bce_f64(rowStart.data_ptr(), col.data_ptr(), rels.data_ptr(), n, nnz, R,
                                                                  X.data_ptr(), r, X.data_ptr(), r, Dt.data_ptr(), r, r, 1.0, inv,
                                                                  dX.data_ptr(), r, stats.data_ptr(), 2, scores.data_ptr(),
                                                                  g.data_ptr(), st), "distmult_bce"), reps)
            grad = event_time(lambda: check(L.hnh_distmult_bce_grad_f64(rowStart.data_ptr(), col.data_ptr(), rels.data_ptr(), n, nnz,
                                                                        R, X.data_ptr(), r, X.data_ptr(), r, Dt.data_ptr(), r, r, 1.0,
                                                                        inv, dX.data_ptr(), r, st), "distmult_bce_grad"), reps)
            fb = base + nnz * 16 + R * r * 8
            gb = base - n * 32 + R * r * 8
            rec.update(kernel_fwd_ms=fwd * 1e3, kernel_fwd_hbm=fb / fwd / HBM, kernel_grad_ms=grad * 1e3, kernel_grad_hbm=gb / grad / HBM,
                       kernel_link_ms=link * 1e3, kernel_link_hbm=base / link / HBM, fwd_over_link=fwd / link)
        # the dD pass through the op's plan: the op with dD minus the op without
        alg = D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(n, n, rows_g, cols_g, rels_np), r, 1)
        H = D.Dense.create(alg.like_A_matrix().shape[0], r)
        H.from_host(np.vstack([X.cpu().numpy(), np.zeros((H.shape[0] - n, r))]))
        Dd = D.Dense.create(R, r)
        Dd.from_host(Dt.cpu().numpy())
        dH, dD = D.Dense.create(*H.shape), D.Dense.create(R, r)
        op_a = timed(lambda: alg.distmult_loss(H, H, Dd, R, 1.0, inv, dH, dH), reps)
        op_ad = timed(lambda: alg.distmult_loss(H, H, Dd, R, 1.0, inv, dH, dH, dD), reps)
        rec.update(op_grad_ms=op_a * 1e3, op_grad_dD_ms=op_ad * 1e3, dD_pass_ms=(op_ad - op_a) * 1e3,
                   dD_over_grad=(op_ad - op_a) / grad if grad else None,
                   dD_pass_hbm=(nnz * (2 * r * 8 + 24)) / max(op_ad - op_a, 1e-12) / HBM)
        if "op" in parts:
            # the torch composition: forward plus backward, autograd
            u, v, rho = torch.from_numpy(rows_g).cuda(), col, rels.long()
            Ht = X.clone().requires_grad_()
            Dtt = Dt.clone().requires_grad_()

            def composed():
                s = (Ht.index_select(0, u) * Dtt.index_select(0, rho) * Ht.index_select(0, v)).sum(1)
                loss = F.binary_cross_entropy_with_logits(s, ones, reduction="mean")
                Ht.grad = Dtt.grad = None
                loss.backward()

            try:
                comp = timed(composed, max(reps // 2, 2))
                rec.update(torch_fwd_bwd_ms=comp * 1e3, op_speedup=comp / op_ad)
            except torch.cuda.OutOfMemoryError:
                rec.update(torch_fwd_bwd_ms=None, torch_note="out of memory")
            torch.cuda.empty_cache()
        del alg, H, dH, dD, Dd
        out(rec)


def train_part(out):
    import numpy as np

    from distributed_sddmm_b200 import driver as D
    from oracle import hnh_oracle as orc
    logM, trials = int(env("TRAIN_LOGM", "16")), int(env("TRIALS", "5"))
    npr_s, npr_t, R = int(env("NPR_S", "16")), int(env("NPR_T", "8")), int(env("R_TRAIN", "8"))
    N = 1 << logM
    rows, cols, _ = orc.er_tuples(logM, npr_s, 0xC0FFEE)
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    alg = D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, rows, cols, ((rows + 3 * cols) % R).astype(np.float64)),
                      TRAIN_LAYERS[0][0], 1)
    net = D.RGCN(alg, TRAIN_LAYERS, num_relations=R)
    rng = np.random.default_rng(2)
    for l, (f, o) in enumerate(TRAIN_LAYERS):
        net.set_param(l, "weight", rng.uniform(-1, 1, (R * f, o)) / np.sqrt(f))
        net.set_param(l, "root", rng.uniform(-1, 1, (f, o)) / np.sqrt(f))
    net.set_input(rng.uniform(-1, 1, net.buffer_shape(0)))
    tr, tc, _ = orc.er_tuples(logM, npr_t, 0xBEEF)
    tr, tc = np.asarray(tr, np.int64), np.asarray(tc, np.int64)
    half = len(tr) // 2
    rel = rng.integers(0, R, len(tr)).astype(np.float64)
    mk = lambda a, b, v: D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, a, b, v), TRAIN_LAYERS[0][0], 1)  # noqa: E731
    a_pos, a_neg = mk(tr[:half], tc[:half], rel[:half]), mk(tr[half:], tc[half:], rel[half:])
    a_link = mk(tr, tc, np.concatenate([np.ones(half), np.zeros(len(tr) - half)]))
    dec = D.DistMultDecoder(net, R)
    dec.set_param("rel", rng.uniform(0.5, 1.5, (R, TRAIN_LAYERS[-1][1])))
    t = D.RelationalLinkTargets(net, a_pos, a_neg, R)
    lt = D.LinkTargets(net, a_link)
    opt, opt2 = D.AdamW(lr=1e-4), D.AdamW(lr=1e-4)
    rel_step = lambda: net.relational_link_train_step(dec, t, opt)  # noqa: E731
    dot_step = lambda: net.link_train_step(lt, opt2)  # noqa: E731
    rel_step(), dot_step()
    tr_rel, tr_dot = [], []
    for _ in range(trials):  # alternate the two
        t0 = time.perf_counter()
        rel_step()
        tr_rel.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        dot_step()
        tr_dot.append(time.perf_counter() - t0)
    a, b = float(np.median(tr_rel)), float(np.median(tr_dot))
    out(dict(part="train", logM=logM, npr_s=npr_s, npr_t=npr_t, R=R, layers=TRAIN_LAYERS, pairs=len(tr),
             relational_step_ms=a * 1e3, link_step_ms=b * 1e3, ratio=a / b))


def main():
    import torch
    if not torch.cuda.is_available():
        sys.exit("distmult_bench.py needs a GPU")
    from distributed_sddmm_b200 import driver as D
    print(json.dumps({"card": card()}), flush=True)
    parts = env("PARTS", "kernels,op,train").split(",")
    D.world_init("self")
    out = lambda rec: print(json.dumps(rec), flush=True)  # noqa: E731
    if "kernels" in parts or "op" in parts:
        kernels_and_op(out, parts)
    if "train" in parts:
        train_part(out)
    D.world_finalize()


if __name__ == "__main__":
    main()
