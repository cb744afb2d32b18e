#!/usr/bin/env python
"""Filtered link ranking on one GPU: the count kernel against the DMMA GEMM that writes the same scores, net.link_rank
against a chunked torch composition, and PyG's per-query loop.  Prints the card name and power limit first, then one
JSON line per measurement.

kernel (Z: KROWS x r, Q: KQUERIES x r, random; r in KWIDTHS): hnh_rank_count_f64 against hnh_dgemm_nt_f64 computing and
  writing the KROWS x KQUERIES score matrix, REPS launches each between CUDA events.  TFLOP/s on 2 rows queries r
  operations, and that rate's share of the data sheet's 67 fp64 TFLOP/s (tensor core, H100 SXM at 700 W).
e2e (a one-layer GraphSAGE, 16 -> r, over an Erdos-Renyi S of 4 draws per row, whose output is the embedding table, and
  a DistMult decoder with random relations): net.link_rank against the torch composition on the same output rows --
  per query chunk the query block z[anchor] * rel[rho], torch.matmul with the embedding table, the filter applied as
  -inf at the excluded (query, node) pairs (their indices built on the host beforehand and not timed), the true score
  gathered, then the > and >= counts summed -- for both directions, each call ending in a synchronise.  Two shapes:
    fb15k: M = 14,541, R = 237, r = 500, 20,466 queries, 310,116 filter triples (FB15k-237's sizes, random triples);
    large: M = 2^20, R = 16, r = 128, 65,536 queries, 262,144 filter triples.
  The queries are drawn from the filter triples.
  The ranks of the two are compared (the GEMMs round differently, so a few ranks near ties may differ).
loop: PyG's compute_mrr loop (tests/link_ranking_oracle.py) on the CPU, per query, over LOOP_QUERIES queries of fb15k.

Environment: PARTS (kernel,e2e,loop), KROWS (131072), KQUERIES (4096), KWIDTHS (128,500), REPS (5), SHAPES
(fb15k,large), LOOP_QUERIES (20)."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_FP64 = 67e12
SHAPES = {"fb15k": dict(M=14541, R=237, r=500, n_q=20466, n_f=310116),
          "large": dict(M=1 << 20, R=16, r=128, n_q=65536, n_f=4 * 65536)}


def env(name, default):
    return os.environ.get(name, default)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


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


def synced(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, res


def kernel(out):
    import torch

    from distributed_sddmm_b200 import check, lib
    L = lib()
    rows, n_q, reps = int(env("KROWS", "131072")), int(env("KQUERIES", "4096")), int(env("REPS", "5"))
    g = torch.Generator(device="cuda").manual_seed(0)
    st = torch.cuda.current_stream().cuda_stream
    for r in (int(x) for x in env("KWIDTHS", "128,500").split(",")):
        Z = torch.randn(rows, r, dtype=torch.float64, device="cuda", generator=g)
        Q = torch.randn(n_q, r, dtype=torch.float64, device="cuda", generator=g)
        s_true = torch.randn(n_q, dtype=torch.float64, device="cuda", generator=g) * r ** 0.5
        counts = torch.zeros(2, n_q, dtype=torch.int64, device="cuda")
        C = torch.empty(rows, n_q, dtype=torch.float64, device="cuda")
        flops = 2.0 * rows * n_q * r
        t_count = event_time(lambda: check(L.hnh_rank_count_f64(Z.data_ptr(), r, rows, Q.data_ptr(), r, n_q, r, s_true.data_ptr(),
                                                                counts[0].data_ptr(), counts[1].data_ptr(), st), "rank_count"), reps)
        t_gemm = event_time(lambda: check(L.hnh_dgemm_nt_f64(C.data_ptr(), Z.data_ptr(), Q.data_ptr(), rows, n_q, r, 0, st), "dgemm_nt"),
                            reps)
        # the counts against the written scores (the same DMMA tiling and k order: equal)
        counts.zero_()
        check(L.hnh_rank_count_f64(Z.data_ptr(), r, rows, Q.data_ptr(), r, n_q, r, s_true.data_ptr(), counts[0].data_ptr(),
                                   counts[1].data_ptr(), st), "rank_count")
        same = bool(torch.equal(counts[0], (C > s_true[None, :]).sum(0)) and torch.equal(counts[1], (C >= s_true[None, :]).sum(0)))
        for name, t in (("hnh_rank_count_f64", t_count), ("hnh_dgemm_nt_f64", t_gemm)):
            out(dict(part="kernel", kernel=name, rows=rows, queries=n_q, r=r, ms=round(t * 1e3, 3), tflops=round(flops / t / 1e12, 2),
                     share_of_67=round(flops / t / PEAK_FP64, 3), score_bytes=0 if name == "hnh_rank_count_f64" else rows * n_q * 8,
                     counts_equal_gemm=same))
        del Z, Q, C


def synthetic(shape, seed=0):
    import numpy as np
    rng = np.random.default_rng(seed)
    M, R, n_q, n_f = (SHAPES[shape][k] for k in ("M", "R", "n_q", "n_f"))
    F = tuple(rng.integers(0, hi, n_f).astype(np.int64) for hi in (M, R, M))
    pick = rng.choice(n_f, min(n_q, n_f), replace=False)
    q = tuple(a[pick] for a in F)
    if n_q > n_f:
        extra = tuple(rng.integers(0, hi, n_q - n_f).astype(np.int64) for hi in (M, R, M))
        q = tuple(np.concatenate([a, b]) for a, b in zip(q, extra))
        F = tuple(np.concatenate([a, b]) for a, b in zip(F, extra))
    return F, q


def excluded_pairs(F, q, M, R, tail):
    """(query, node) pairs removed from the candidates: the true entity and the known ones (host, numpy)."""
    import numpy as np
    h, rho, t = q
    fa, fr, fb = (F[0], F[1], F[2]) if tail else (F[2], F[1], F[0])
    anchor, target = (h, t) if tail else (t, h)
    key = fa * R + fr
    order = np.argsort(key, kind="stable")
    ks, vs = key[order], fb[order]
    qk = anchor * R + rho
    lo, hi = np.searchsorted(ks, qk, "left"), np.searchsorted(ks, qk, "right")
    cnt = hi - lo
    qi = np.repeat(np.arange(len(qk)), cnt)
    starts = np.repeat(lo - np.concatenate([[0], np.cumsum(cnt)[:-1]]), cnt)
    vi = vs[np.arange(cnt.sum()) + starts]
    return np.concatenate([qi, np.arange(len(qk))]), np.concatenate([vi, target])


def torch_ranks(z, rel, q, pairs, chunk):
    import torch
    h, rho, t = (torch.as_tensor(a, device="cuda") for a in q)
    res = []
    for tail, (pq, pv) in zip((True, False), pairs):
        anchor, target = (h, t) if tail else (t, h)
        gt, ge = torch.empty(len(h), dtype=torch.int64, device="cuda"), torch.empty(len(h), dtype=torch.int64, device="cuda")
        for c0 in range(0, len(h), chunk):
            c1 = min(c0 + chunk, len(h))
            Qc = z[anchor[c0:c1]] * rel[rho[c0:c1]]
            S = Qc @ z.T
            true = S[torch.arange(c1 - c0, device="cuda"), target[c0:c1]]
            lo, hi = torch.searchsorted(pq, c0), torch.searchsorted(pq, c1)
            S[pq[lo:hi] - c0, pv[lo:hi]] = -torch.inf
            gt[c0:c1] = (S > true[:, None]).sum(1)
            ge[c0:c1] = (S >= true[:, None]).sum(1)
            del S
        res.append(((gt + 1) + (ge + 1)).double() / 2)
    return res


def e2e(out):
    import numpy as np
    import torch

    from distributed_sddmm_b200 import driver as D
    for shape in env("SHAPES", "fb15k,large").split(","):
        M, R, r, n_q, n_f = (SHAPES[shape][k] for k in ("M", "R", "r", "n_q", "n_f"))
        F, q = synthetic(shape)
        rng = np.random.default_rng(1)
        rows, cols = rng.integers(0, M, 4 * M), rng.integers(0, M, 4 * M)
        alg = D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(M, M, rows, cols, np.ones(4 * M)), 16, 1)
        net = D.GraphSAGE(alg, [(16, r)], aggr="mean")
        net.set_param(0, "neigh", rng.uniform(-1, 1, (16, r)) / 4)
        net.set_param(0, "root", rng.uniform(-1, 1, (16, r)) / 4)
        net.set_input(rng.uniform(-1, 1, net.buffer_shape(0)))
        dec = D.DistMultDecoder(net, R)
        dec.set_param("rel", rng.uniform(-1, 1, (R, r)))
        t0 = time.perf_counter()
        ranking = D.LinkRanking(net, F, R)
        t_build = time.perf_counter() - t0
        net.link_rank(ranking, tuple(a[:64] for a in q), decoder=dec)  # warm-up
        t_lib, res = synced(lambda: net.link_rank(ranking, q, decoder=dec))
        z = torch.as_tensor(net.buffer(1)[:M], device="cuda")
        rel = torch.as_tensor(dec.param("rel"), device="cuda")
        pairs = []
        for tail in (True, False):
            pq, pv = excluded_pairs(F, q, M, R, tail)
            o = np.argsort(pq, kind="stable")
            pairs.append((torch.as_tensor(pq[o], device="cuda"), torch.as_tensor(pv[o], device="cuda")))
        chunk = max(64, min(n_q, (1 << 31) // (8 * M)))  # a 2 GiB score block
        torch_ranks(z, rel, tuple(a[:64] for a in q), [(p[0][:0], p[1][:0]) for p in pairs], chunk)  # warm-up
        t_torch, tr = synced(lambda: torch_ranks(z, rel, q, pairs, chunk))
        diff_t = np.abs(tr[0].cpu().numpy() - res.tail_ranks)
        diff_h = np.abs(tr[1].cpu().numpy() - res.head_ranks)
        flops = 2 * 2.0 * n_q * M * r
        out(dict(part="e2e", shape=shape, M=M, R=R, r=r, queries=n_q, filter=len(F[0]), link_rank_s=round(t_lib, 3),
                 torch_s=round(t_torch, 3), speedup=round(t_torch / t_lib, 2), filter_build_s=round(t_build, 3),
                 link_rank_tflops=round(flops / t_lib / 1e12, 2), mrr=res.mrr, hits10=res.hits_at(10),
                 ranks_differing=int((diff_t > 0).sum() + (diff_h > 0).sum()), max_rank_diff=float(max(diff_t.max(), diff_h.max())),
                 torch_chunk=chunk))
        del net, alg, dec, ranking, z


def loop(out):
    import numpy as np

    from tests import link_ranking_oracle as lro
    n = int(env("LOOP_QUERIES", "20"))
    s = SHAPES["fb15k"]
    F, q = synthetic("fb15k")
    rng = np.random.default_rng(2)
    z, rel = rng.standard_normal((s["M"], s["r"])), rng.standard_normal((s["R"], s["r"]))
    t0 = time.perf_counter()
    lro.compute_mrr_loop(z, lro.decoder_of(rel), tuple(a[:n] for a in q), [F], s["M"])
    t = (time.perf_counter() - t0) / n
    out(dict(part="loop", shape="fb15k", device="cpu", queries=n, ms_per_query=round(t * 1e3, 2),
             projected_s=round(t * s["n_q"], 1)))


def main():
    import torch

    from distributed_sddmm_b200 import driver as D
    if not torch.cuda.is_available():
        sys.exit("link_ranking_bench: no GPU")
    print(json.dumps({"card": card()}), flush=True)
    parts = env("PARTS", "kernel,e2e,loop").split(",")
    D.world_init("self")
    out = lambda rec: print(json.dumps(rec), flush=True)  # noqa: E731
    if "kernel" in parts:
        kernel(out)
    if "e2e" in parts:
        e2e(out)
    if "loop" in parts:
        loop(out)
    D.world_finalize()


if __name__ == "__main__":
    main()
