#!/usr/bin/env python
"""CUDA-event time of fused sparse attention on one GPU, at the kernel level and at the op level.

Kernels, on the A-order CSR block of an Erdos-Renyi 2^LOGM x 2^LOGM S with NPR draws per row under ALG at p = 1
(15d_fusion1: 2^20 rows and 33 553 937 entries at the defaults) and, for the key-side gradient, the B-order block,
at each d of WIDTHS: the step (hnh_sparse_attention_step_f64), the finish, and the two gradients, beside the
overwrite-form SDDMM (hnh_sddmm_f64 with HNH_FLAG_BETA0) and the accumulating SpMM (hnh_spmm_f64) on the same block.
Algorithmic bytes per call (int64 indices, fp64 values; a gathered row counted once per entry, as if no cache held it):
    sddmm (overwrite)  nnz (8 col + 8 value + 8 d gathered) + rows (8 row start + 8 d row side)
    spmm (accumulate)  nnz (8 col + 8 value + 8 d gathered) + rows (8 row start + 16 d output read and write)
    step               nnz (8 col + 16 d K and V) + rows (8 row start + 8 d Q + 16 d acc read and write + 32 m, s)
    finish             rows (24 d + 32)
    grad_q             nnz (8 col + 16 d K and V) + rows (8 row start + 16 d Q, dZ + 16 L, t + 16 d dQ read and write)
    grad_kv            nnz (8 col + 16 d Q and dZ + 16 L, t) + rows (8 row start + 16 d K, V + 32 d dK, dV read and write)
set against the H100 SXM's 3.35 TB/s.  Op level, one head of width d: Algorithm.sparse_attention and
sparse_attention_backward beside the composed public ops -- forward: scaled sddmmA, edge_softmax, spmmA; backward:
alpha in both orders (2 scaled SDDMMs, 2 softmaxes), dalpha in both orders (2 SDDMMs), 2 softmax backwards and the
dV, dQ, dK SpMMs -- with the composed path's first edge_softmax per order (which builds its row grouping) timed
separately, and the largest relative difference between the two.  Prints the card name and power limit, then one
JSON line per measurement.

Attention dropout at DROPOUT (0.1): each of the three dropout kernels (hnh_sparse_attention_*_dropout_f64) beside its
kernel without dropout on the same block and operands, the two timed in alternation ROUNDS (5) times, REPS launches
each, with the median of each and their ratio; then Algorithm.sparse_attention and sparse_attention_backward with and
without dropout, alternated the same way.

Additive score bias (PARTS=bias): each of the three bias kernels (hnh_sparse_attention_*_bias_f64, p = 0, a bias
uniform in [-1, 1), the gradients writing dbias) beside its kernel without bias, alternated the same way; the two
gradient kernels with and without the dbias write; then Algorithm.sparse_attention and sparse_attention_backward
(writing both dbias vectors) with and without a bias.  The bias adds 8 bytes read per entry, and dbias 16 more (read
and write), to the byte counts above.
Edge features (PARTS=edge): each of the three edge kernels (hnh_sparse_attention_*_edge_f64, p = 0, no bias, E
uniform in [-1, 1), grad_q writing dE) beside its kernel without E, alternated the same way, with the ratio of their
bytes/s; then Algorithm.sparse_attention and sparse_attention_backward (writing dE) with and without E.  E adds 8d
bytes read per entry to the step and to grad_kv, and 16d (E read, dE written) to grad_q; a gathered row still counts
once per entry.  E, its B-order copy and dE take 3 x 8 d bytes per entry (51 GB at 2^20 rows, 32 per row and d = 64),
so run this part at WIDTHS=32,64.  PARTS (kernels,ops,dropout; also bias, edge) picks the sections.
Environment: LOGM (20), NPR (32), WIDTHS (128,256), ALG (15d_fusion1), REPS (20), DROPOUT (0.1), ROUNDS (5), PARTS."""
import json
import math
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
widths = [int(x) for x in os.environ.get("WIDTHS", "128,256").split(",")]
alg_name = os.environ.get("ALG", "15d_fusion1")
reps = int(os.environ.get("REPS", "20"))
dropout = float(os.environ.get("DROPOUT", "0.1"))
rounds = int(os.environ.get("ROUNDS", "5"))
parts = os.environ.get("PARTS", "kernels,ops,dropout").split(",")
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


def timed_op(call):
    """The same on the library's compute stream, where the operations run."""
    call()
    D.timer_start()
    for _ in range(reps):
        call()
    return D.timer_stop() / reps


def once_op(call):
    D.timer_start()
    call()
    return D.timer_stop()


def report(kernel, d, ms, nbytes=None, **extra):
    rec = dict(kernel=kernel, logM=logM, nnz_per_row=npr, d=d, ms_per_call=round(ms, 4), **extra)
    if nbytes:
        rec.update(min_bytes=nbytes, tb_per_s=round(nbytes / (ms * 1e-3) / 1e12, 3),
                   share_of_3_35_tb_s=round(nbytes / (ms * 1e-3) / HBM, 3))
    print(json.dumps(rec), flush=True)
    return ms


def block(alg, which):
    blocks = [b for b in alg.blocks(which) if b is not None]
    assert len(blocks) == 1, "one local block at p = 1"
    b = blocks[0]
    return int(b["rows"]), len(b["col_idx"]), torch.from_numpy(b["rowStart"]).to(dev), torch.from_numpy(b["col_idx"]).to(dev)


def kernels(alg, d):
    # fusion 1 keeps the A order in ST's block (S-rows as stored rows) and the B order in S's
    a_blk, b_blk = ("ST", "S") if alg_name == "15d_fusion1" else ("S", "ST")
    rows, nnz, rs, ci = block(alg, a_blk)
    rowsT, nnzT, rsT, ciT = block(alg, b_blk)
    g = torch.Generator(device=dev).manual_seed(1)
    Q, K, V, dZ = (torch.rand((max(rows, rowsT), d), generator=g, **f64) * 2 - 1 for _ in range(4))
    acc, dQ, dK, dV = (torch.zeros((max(rows, rowsT), d), **f64) for _ in range(4))
    ms_ = torch.zeros((rows, 2), **f64)
    Lt = torch.zeros((max(rows, rowsT), 2), **f64)
    values = torch.rand(nnz, generator=g, **f64)
    out = torch.empty(nnz, **f64)
    scale = 1 / math.sqrt(d)
    p = lambda t: t.data_ptr()  # noqa: E731
    sddmm = report("sddmm_overwrite", d, timed(lambda: D.check(L.hnh_sddmm_f64(
        p(rs), p(ci), p(out), rows, nnz, p(Q), p(K), d, BETA0, st))), nnz * (16 + 8 * d) + rows * (8 + 8 * d))
    spmm = report("spmm_accumulate", d, timed(lambda: D.check(L.hnh_spmm_f64(
        p(rs), p(ci), p(values), rows, nnz, p(V), p(acc), d, 0, st))), nnz * (16 + 8 * d) + rows * (8 + 16 * d))
    base = sddmm + spmm

    def step():
        D.check(L.hnh_sparse_attention_step_f64(p(rs), p(ci), rows, nnz, d, p(Q), d, p(K), d, p(V), d, scale, p(acc), d,
                                                p(ms_), 2, p(ms_) + 8, 2, st))
    acc.zero_()
    ms_.zero_()
    st_ms = report("step", d, timed(step), nnz * (8 + 16 * d) + rows * (8 + 24 * d + 32))
    finish = report("finish", d, timed(lambda: D.check(L.hnh_sparse_attention_finish_f64(
        rows, d, p(acc), d, p(ms_), 2, p(ms_) + 8, 2, p(dQ), d, p(Lt), 2, st))), rows * (24 * d + 32))
    gq = report("grad_q", d, timed(lambda: D.check(L.hnh_sparse_attention_grad_q_f64(
        p(rs), p(ci), rows, nnz, d, p(Q), d, p(dZ), d, p(Lt), 2, p(Lt) + 8, 2, p(K), d, p(V), d, scale, p(dQ), d, st))),
        nnz * (8 + 16 * d) + rows * (8 + 32 * d + 16))
    gkv = report("grad_kv", d, timed(lambda: D.check(L.hnh_sparse_attention_grad_kv_f64(
        p(rsT), p(ciT), rowsT, nnzT, d, p(K), d, p(V), d, p(Q), d, p(dZ), d, p(Lt), 2, p(Lt) + 8, 2, scale, p(dK), d, p(dV), d,
        st))), nnzT * (24 + 16 * d) + rowsT * (8 + 48 * d))
    print(json.dumps(dict(d=d, entries=nnz, rows=rows, step_over_sddmm_plus_spmm=round(st_ms / base, 3),
                          step_plus_finish_over_sddmm_plus_spmm=round((st_ms + finish) / base, 3),
                          grad_q_over_sddmm_plus_spmm=round(gq / base, 3),
                          grad_kv_over_sddmm_plus_spmm=round(gkv / base, 3))), flush=True)


def rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


def ops(d):
    alg = D.Algorithm(alg_name, S, d, 1)
    dims = alg.dims
    rng = np.random.default_rng(SEED)
    mats = {}
    for name, which in (("Q", "A"), ("dZ", "A"), ("K", "B"), ("V", "B")):
        m = alg.like_A_matrix() if which == "A" else alg.like_B_matrix()
        m.from_host(rng.uniform(-1, 1, m.shape))
        mats[name] = m
    Q, K, V, dZ = (mats[k] for k in ("Q", "K", "V", "dZ"))
    Z, dQ, dK, dV = alg.like_A_matrix(), alg.like_A_matrix(), alg.like_B_matrix(), alg.like_B_matrix()
    Lm = D.Dense.create(dims.localArows, 1)
    scale = 1 / math.sqrt(d)
    fwd = report("op_fused_forward", d, timed_op(lambda: alg.sparse_attention(Q, K, V, Z, Lm)))
    bwd = report("op_fused_backward", d, timed_op(lambda: alg.sparse_attention_backward(Q, K, V, Z, Lm, dZ, dQ, dK, dV)))
    # composed: the first edge_softmax per order builds its row grouping
    sA, sB, oneA, oneB = alg.like_S_values(scale), alg.like_ST_values(scale), alg.like_S_values(1.0), alg.like_ST_values(1.0)
    xA, xB, gA, gB = alg.like_S_values(), alg.like_ST_values(), alg.like_S_values(), alg.like_ST_values()
    Zc, dQc, dKc, dVc = alg.like_A_matrix(), alg.like_A_matrix(), alg.like_B_matrix(), alg.like_B_matrix()
    alg.sddmmA(Q, K, sA, xA)
    alg.sddmmB(Q, K, sB, xB)
    plan_a = once_op(lambda: alg.edge_softmax(xA, "A"))
    plan_b = once_op(lambda: alg.edge_softmax(xB, "B"))

    def c_forward():
        alg.sddmmA(Q, K, sA, xA)
        alg.edge_softmax(xA, "A")
        alg.spmmA(Zc, V, xA)

    def c_backward():
        alg.sddmmA(Q, K, sA, xA)
        alg.edge_softmax(xA, "A")
        alg.sddmmB(Q, K, sB, xB)
        alg.edge_softmax(xB, "B")
        alg.sddmmA(dZ, V, oneA, gA)
        alg.sddmmB(dZ, V, oneB, gB)
        alg.edge_softmax_backward(xA, gA, "A")
        alg.edge_softmax_backward(xB, gB, "B")
        alg.spmmB(dZ, dVc, xB)
        alg.spmmA(dQc, K, gA)
        alg.spmmB(Q, dKc, gB)

    cf = report("op_composed_forward", d, timed_op(c_forward), first_edge_softmax_ms=dict(A=round(plan_a, 3), B=round(plan_b, 3)))
    cb = report("op_composed_backward", d, timed_op(c_backward))
    # the composed dQ and dK leave out the final factor scale
    agree = dict(Z=rel(Z.to_host(), Zc.to_host()), dV=rel(dV.to_host(), dVc.to_host()),
                 dQ=rel(dQ.to_host(), scale * dQc.to_host()), dK=rel(dK.to_host(), scale * dKc.to_host()))
    print(json.dumps(dict(d=d, forward_fused_over_composed=round(fwd / cf, 3), backward_fused_over_composed=round(bwd / cb, 3),
                          max_rel_difference=agree, agree_within_1e_12=all(v < 1e-12 for v in agree.values()))), flush=True)
    del alg


def alternate(name, d, plain, dropped, timer=timed, nbytes=None):
    """plain and dropped timed in turn `rounds` times; their medians and ratio."""
    a, b = [], []
    for _ in range(rounds):
        a.append(timer(plain))
        b.append(timer(dropped))
    ma, mb = float(np.median(a)), float(np.median(b))
    report(name, d, ma, nbytes, dropout=0.0, spread=[round(min(a), 4), round(max(a), 4)])
    report(name + "_dropout", d, mb, nbytes, dropout=dropout, spread=[round(min(b), 4), round(max(b), 4)])
    return mb / ma


def dropout_kernels(alg, d):
    a_blk, b_blk = ("ST", "S") if alg_name == "15d_fusion1" else ("S", "ST")
    rows, nnz, rs, ci = block(alg, a_blk)
    rowsT, nnzT, rsT, ciT = block(alg, b_blk)
    g = torch.Generator(device=dev).manual_seed(1)
    n = max(rows, rowsT)
    Q, K, V, dZ = (torch.rand((n, d), generator=g, **f64) * 2 - 1 for _ in range(4))
    acc, dQ, dK, dV = (torch.zeros((n, d), **f64) for _ in range(4))
    ms_ = torch.zeros((rows, 2), **f64)
    Lt = torch.rand((n, 2), generator=g, **f64) + 4  # L, t: a plausible log-sum-exp of 32 entries, and <dZ, Z>
    scale = 1 / math.sqrt(d)
    p = lambda t: t.data_ptr()  # noqa: E731
    drop = (dropout, SEED, 0, 0)

    def step(*dr):
        fn = L.hnh_sparse_attention_step_dropout_f64 if dr else L.hnh_sparse_attention_step_f64
        D.check(fn(p(rs), p(ci), rows, nnz, d, p(Q), d, p(K), d, p(V), d, scale, p(acc), d, p(ms_), 2, p(ms_) + 8, 2, *dr, st))

    def grad_q(*dr):
        fn = L.hnh_sparse_attention_grad_q_dropout_f64 if dr else L.hnh_sparse_attention_grad_q_f64
        D.check(fn(p(rs), p(ci), rows, nnz, d, p(Q), d, p(dZ), d, p(Lt), 2, p(Lt) + 8, 2, p(K), d, p(V), d, scale, p(dQ), d,
                   *dr, st))

    def grad_kv(*dr):
        fn = L.hnh_sparse_attention_grad_kv_dropout_f64 if dr else L.hnh_sparse_attention_grad_kv_f64
        D.check(fn(p(rsT), p(ciT), rowsT, nnzT, d, p(K), d, p(V), d, p(Q), d, p(dZ), d, p(Lt), 2, p(Lt) + 8, 2, scale, p(dK), d,
                   p(dV), d, *dr, st))

    ratios = {}
    for name, fn, nbytes in (("step", step, nnz * (8 + 16 * d) + rows * (8 + 24 * d + 32)),
                             ("grad_q", grad_q, nnz * (8 + 16 * d) + rows * (8 + 32 * d + 16)),
                             ("grad_kv", grad_kv, nnzT * (24 + 16 * d) + rowsT * (8 + 48 * d))):
        ratios[name] = round(alternate(name, d, fn, lambda fn=fn: fn(*drop), nbytes=nbytes), 3)
    print(json.dumps(dict(d=d, dropout=dropout, dropout_kernel_over_kernel=ratios)), flush=True)


def dropout_ops(d):
    alg = D.Algorithm(alg_name, S, d, 1)
    dims = alg.dims
    rng = np.random.default_rng(SEED)
    Q, dZ = (alg.like_A_matrix() for _ in range(2))
    K, V = (alg.like_B_matrix() for _ in range(2))
    for m in (Q, dZ, K, V):
        m.from_host(rng.uniform(-1, 1, m.shape))
    Z, dQ, dK, dV = alg.like_A_matrix(), alg.like_A_matrix(), alg.like_B_matrix(), alg.like_B_matrix()
    Lm = D.Dense.create(dims.localArows, 1)
    kw = dict(dropout=dropout, seed=SEED)
    fwd = alternate("op_fused_forward", d, lambda: alg.sparse_attention(Q, K, V, Z, Lm),
                    lambda: alg.sparse_attention(Q, K, V, Z, Lm, **kw), timer=timed_op)
    alg.sparse_attention(Q, K, V, Z, Lm, **kw)
    bwd = alternate("op_fused_backward", d, lambda: alg.sparse_attention_backward(Q, K, V, Z, Lm, dZ, dQ, dK, dV),
                    lambda: alg.sparse_attention_backward(Q, K, V, Z, Lm, dZ, dQ, dK, dV, **kw), timer=timed_op)
    print(json.dumps(dict(d=d, dropout=dropout, forward_dropout_over_forward=round(fwd, 3),
                          backward_dropout_over_backward=round(bwd, 3))), flush=True)
    del alg


def alternate_pair(names, d, calls, timer=timed, nbytes=(None, None)):
    """calls[0] and calls[1] timed in turn `rounds` times, reported under names[0] and names[1]; the ratio of their
    medians (second over first)."""
    t = ([], [])
    for _ in range(rounds):
        for i in (0, 1):
            t[i].append(timer(calls[i]))
    med = [float(np.median(x)) for x in t]
    for i in (0, 1):
        report(names[i], d, med[i], nbytes[i], spread=[round(min(t[i]), 4), round(max(t[i]), 4)])
    return med[1] / med[0]


def bias_kernels(alg, d):
    a_blk, b_blk = ("ST", "S") if alg_name == "15d_fusion1" else ("S", "ST")
    rows, nnz, rs, ci = block(alg, a_blk)
    rowsT, nnzT, rsT, ciT = block(alg, b_blk)
    g = torch.Generator(device=dev).manual_seed(1)
    n = max(rows, rowsT)
    Q, K, V, dZ = (torch.rand((n, d), generator=g, **f64) * 2 - 1 for _ in range(4))
    acc, dQ, dK, dV = (torch.zeros((n, d), **f64) for _ in range(4))
    ms_ = torch.zeros((rows, 2), **f64)
    Lt = torch.rand((n, 2), generator=g, **f64) + 4  # L, t: a plausible log-sum-exp of 32 entries, and <dZ, Z>
    bA, bB = torch.rand(nnz, generator=g, **f64) * 2 - 1, torch.rand(nnzT, generator=g, **f64) * 2 - 1
    dbA, dbB = torch.zeros(nnz, **f64), torch.zeros(nnzT, **f64)
    scale = 1 / math.sqrt(d)
    p = lambda t: t.data_ptr()  # noqa: E731
    nob = (0.0, SEED, 0, 0)

    def step(b=False):
        if b:
            D.check(L.hnh_sparse_attention_step_bias_f64(p(rs), p(ci), rows, nnz, d, p(Q), d, p(K), d, p(V), d, scale, p(acc), d,
                                                         p(ms_), 2, p(ms_) + 8, 2, *nob, p(bA), st))
        else:
            D.check(L.hnh_sparse_attention_step_f64(p(rs), p(ci), rows, nnz, d, p(Q), d, p(K), d, p(V), d, scale, p(acc), d,
                                                    p(ms_), 2, p(ms_) + 8, 2, st))

    def grad_q(b=False, db=True):
        args = (p(rs), p(ci), rows, nnz, d, p(Q), d, p(dZ), d, p(Lt), 2, p(Lt) + 8, 2, p(K), d, p(V), d, scale, p(dQ), d)
        if b:
            D.check(L.hnh_sparse_attention_grad_q_bias_f64(*args, *nob, p(bA), p(dbA) if db else None, st))
        else:
            D.check(L.hnh_sparse_attention_grad_q_f64(*args, st))

    def grad_kv(b=False, db=True):
        args = (p(rsT), p(ciT), rowsT, nnzT, d, p(K), d, p(V), d, p(Q), d, p(dZ), d, p(Lt), 2, p(Lt) + 8, 2, scale, p(dK), d,
                p(dV), d)
        if b:
            D.check(L.hnh_sparse_attention_grad_kv_bias_f64(*args, *nob, p(bB), p(dbB) if db else None, st))
        else:
            D.check(L.hnh_sparse_attention_grad_kv_f64(*args, st))

    ratios = {}
    for name, fn, nbytes, nb, with_db in (
            ("step", step, nnz * (8 + 16 * d) + rows * (8 + 24 * d + 32), nnz * 8, False),
            ("grad_q", grad_q, nnz * (8 + 16 * d) + rows * (8 + 32 * d + 16), nnz * 24, True),
            ("grad_kv", grad_kv, nnzT * (24 + 16 * d) + rowsT * (8 + 48 * d), nnzT * 24, True)):
        ratios[name] = round(alternate_pair((name, name + "_bias"), d, (fn, lambda fn=fn: fn(True)),
                                            nbytes=(nbytes, nbytes + nb)), 3)
        if with_db:
            ratios[name + "_dbias_write"] = round(alternate_pair((name + "_bias_no_dbias", name + "_bias"), d,
                                                                 (lambda fn=fn: fn(True, False), lambda fn=fn: fn(True))), 3)
    print(json.dumps(dict(d=d, bias_kernel_over_kernel=ratios)), flush=True)


def bias_ops(d):
    alg = D.Algorithm(alg_name, S, d, 1)
    dims = alg.dims
    rng = np.random.default_rng(SEED)
    Q, dZ = (alg.like_A_matrix() for _ in range(2))
    K, V = (alg.like_B_matrix() for _ in range(2))
    for m in (Q, dZ, K, V):
        m.from_host(rng.uniform(-1, 1, m.shape))
    Z, dQ, dK, dV = alg.like_A_matrix(), alg.like_A_matrix(), alg.like_B_matrix(), alg.like_B_matrix()
    Lm = D.Dense.create(dims.localArows, 1)
    bA, bB = alg.like_S_values(), alg.like_ST_values()
    rA, cA = alg.entry_coordinates("A")
    rB, cB = alg.entry_coordinates("B")
    bA.from_host(np.sin(0.37 * rA + 1.3 * cA))
    bB.from_host(np.sin(0.37 * rB + 1.3 * cB))
    dbA, dbB = D.Vec.create(0), D.Vec.create(0)
    fwd = alternate_pair(("op_fused_forward", "op_fused_forward_bias"), d,
                         (lambda: alg.sparse_attention(Q, K, V, Z, Lm), lambda: alg.sparse_attention(Q, K, V, Z, Lm, bias=bA)),
                         timer=timed_op)
    alg.sparse_attention(Q, K, V, Z, Lm, bias=bA)
    bwd = alternate_pair(("op_fused_backward", "op_fused_backward_bias"), d,
                         (lambda: alg.sparse_attention_backward(Q, K, V, Z, Lm, dZ, dQ, dK, dV),
                          lambda: alg.sparse_attention_backward(Q, K, V, Z, Lm, dZ, dQ, dK, dV, bias=bA, bias_B=bB, dbias=dbA,
                                                                dbias_B=dbB)), timer=timed_op)
    print(json.dumps(dict(d=d, forward_bias_over_forward=round(fwd, 3), backward_bias_over_backward=round(bwd, 3))),
          flush=True)
    del alg


def edge_kernels(alg, d):
    a_blk, b_blk = ("ST", "S") if alg_name == "15d_fusion1" else ("S", "ST")
    rows, nnz, rs, ci = block(alg, a_blk)
    rowsT, nnzT, rsT, ciT = block(alg, b_blk)
    g = torch.Generator(device=dev).manual_seed(1)
    n = max(rows, rowsT)
    Q, K, V, dZ = (torch.rand((n, d), generator=g, **f64) * 2 - 1 for _ in range(4))
    acc, dQ, dK, dV = (torch.zeros((n, d), **f64) for _ in range(4))
    ms_ = torch.zeros((rows, 2), **f64)
    Lt = torch.rand((n, 2), generator=g, **f64) + 4  # L, t: a plausible log-sum-exp of 32 entries, and <dZ, Z>
    EA, EB = torch.rand((nnz, d), generator=g, **f64) * 2 - 1, torch.rand((nnzT, d), generator=g, **f64) * 2 - 1
    dE = torch.zeros((nnz, d), **f64)
    scale = 1 / math.sqrt(d)
    p = lambda t: t.data_ptr()  # noqa: E731
    noe = (0.0, SEED, 0, 0, None)

    def step(e=False):
        args = (p(rs), p(ci), rows, nnz, d, p(Q), d, p(K), d, p(V), d, scale, p(acc), d, p(ms_), 2, p(ms_) + 8, 2)
        if e:
            D.check(L.hnh_sparse_attention_step_edge_f64(*args, *noe, p(EA), d, st))
        else:
            D.check(L.hnh_sparse_attention_step_f64(*args, st))

    def grad_q(e=False):
        args = (p(rs), p(ci), rows, nnz, d, p(Q), d, p(dZ), d, p(Lt), 2, p(Lt) + 8, 2, p(K), d, p(V), d, scale, p(dQ), d)
        if e:
            D.check(L.hnh_sparse_attention_grad_q_edge_f64(*args, *noe, None, p(EA), d, p(dE), d, st))
        else:
            D.check(L.hnh_sparse_attention_grad_q_f64(*args, st))

    def grad_kv(e=False):
        args = (p(rsT), p(ciT), rowsT, nnzT, d, p(K), d, p(V), d, p(Q), d, p(dZ), d, p(Lt), 2, p(Lt) + 8, 2, scale, p(dK), d,
                p(dV), d)
        if e:
            D.check(L.hnh_sparse_attention_grad_kv_edge_f64(*args, *noe, None, p(EB), d, st))
        else:
            D.check(L.hnh_sparse_attention_grad_kv_f64(*args, st))

    time_ratio, rate_ratio = {}, {}
    for name, fn, nbytes, ne in (("step", step, nnz * (8 + 16 * d) + rows * (8 + 24 * d + 32), nnz * 8 * d),
                                 ("grad_q", grad_q, nnz * (8 + 16 * d) + rows * (8 + 32 * d + 16), nnz * 16 * d),
                                 ("grad_kv", grad_kv, nnzT * (24 + 16 * d) + rowsT * (8 + 48 * d), nnzT * 8 * d)):
        r = alternate_pair((name, name + "_edge"), d, (fn, lambda fn=fn: fn(True)), nbytes=(nbytes, nbytes + ne))
        time_ratio[name] = round(r, 3)
        rate_ratio[name] = round((nbytes + ne) / nbytes / r, 3)
    print(json.dumps(dict(d=d, entries=nnz, edge_kernel_over_kernel_time=time_ratio,
                          edge_kernel_over_kernel_bytes_per_s=rate_ratio)), flush=True)


def edge_ops(d):
    alg = D.Algorithm(alg_name, S, d, 1)
    dims = alg.dims
    rng = np.random.default_rng(SEED)
    Q, dZ = (alg.like_A_matrix() for _ in range(2))
    K, V = (alg.like_B_matrix() for _ in range(2))
    for m in (Q, dZ, K, V):
        m.from_host(rng.uniform(-1, 1, m.shape))
    Z, dQ, dK, dV = alg.like_A_matrix(), alg.like_A_matrix(), alg.like_B_matrix(), alg.like_B_matrix()
    Lm = D.Dense.create(dims.localArows, 1)
    edges = []
    for mode in ("A", "B"):
        r_, c_ = alg.entry_coordinates(mode)
        e = D.Dense.create(len(r_), d)
        e.from_host(np.cos(0.31 * r_[:, None] + 0.73 * c_[:, None] + 0.45 * np.arange(d)[None, :]))
        edges.append(e)
        del r_, c_
    dE = D.Dense.create(1, 1)
    fwd = alternate_pair(("op_fused_forward", "op_fused_forward_edge"), d,
                         (lambda: alg.sparse_attention(Q, K, V, Z, Lm), lambda: alg.sparse_attention(Q, K, V, Z, Lm, edge=edges[0])),
                         timer=timed_op)
    alg.sparse_attention(Q, K, V, Z, Lm, edge=edges[0])
    bwd = alternate_pair(("op_fused_backward", "op_fused_backward_edge"), d,
                         (lambda: alg.sparse_attention_backward(Q, K, V, Z, Lm, dZ, dQ, dK, dV),
                          lambda: alg.sparse_attention_backward(Q, K, V, Z, Lm, dZ, dQ, dK, dV, edge=edges[0], edge_B=edges[1],
                                                                dedge=dE)), timer=timed_op)
    print(json.dumps(dict(d=d, forward_edge_over_forward=round(fwd, 3), backward_edge_over_backward=round(bwd, 3))),
          flush=True)
    del alg


for d in widths:
    alg = D.Algorithm(alg_name, S, d, 1)
    if "kernels" in parts:
        kernels(alg, d)
    if "dropout" in parts:
        dropout_kernels(alg, d)
    if "bias" in parts:
        bias_kernels(alg, d)
    if "edge" in parts:
        edge_kernels(alg, d)
    del alg
    torch.cuda.empty_cache()
    if "ops" in parts:
        ops(d)
    if "dropout" in parts:
        dropout_ops(d)
    if "bias" in parts:
        bias_ops(d)
    if "edge" in parts:
        edge_ops(d)
D.world_finalize()
