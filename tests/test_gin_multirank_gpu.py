"""GIN, GINE and edge-ReLU aggregation on several ranks on the GPU (tests/mp_gin_worker.py), at p = 2 and 4 on the 1.5D
dense shift with replication reuse at c = 1 and 2 and with local kernel fusion at c = 1: the op's A, dX and dE on integer
inputs where X_v + E_i == 0 happens; the model's output, input gradient and parameter gradients (eps and the edge
projection included) against tests/gin_oracle.py's per-edge model on the global graph, row by row; node train steps
against torch AdamW; repeats, parameter gradients and trained parameters bit-identical on every rank; and HNH_E_INVALID
on every rank for the 1.5D sparse shift and for local kernel fusion at c = 2, where rows are not full.

Ranks share cuda:0 over the gloo-backed transport unless there is one GPU per rank (then NCCL)."""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from tests import gin_oracle as go
from tests.mp_gin_worker import LAYERS, global_graph, global_inputs
from tests.mp_util import ROOT, free_port

pytestmark = pytest.mark.gpu

LAYOUTS = [("15d_fusion1", 1), ("15d_fusion1", 2), ("15d_fusion2", 1)]


def case(model, alg, c, logM=7, seed=0xC0FFEE + 433, **kw):
    name = f"{model}_{alg}_c{c}_" + "_".join(f"{k}{v}" for k, v in sorted(kw.items()))
    return dict(name=name, model=model, alg=alg, c=c, logM=logM, seed=seed, **kw)


CASES = {
    p: [case("op", a, c, f=f) for a, c in LAYOUTS for f in (8, 300)]
    + [case("gin", a, c, edge_dim=e) for a, c in LAYOUTS for e in (0, 3)]
    + [case("train", a, c, edge_dim=e) for a, c in LAYOUTS for e in (0, 3)]
    + [case("op", "15d_sparse", 1, f=8, expect="not defined"), case("op", "15d_fusion2", 2, f=8, expect="not defined"),
       case("gin", "15d_sparse", 1, edge_dim=3, expect="not defined"),
       case("gin", "15d_fusion2", 2, edge_dim=0, expect="not defined")]
    for p in (2, 4)
}


def run(nproc, cases, timeout=900):
    """Returns {case name: [per-rank dict]}."""
    transport = "nccl" if torch.cuda.device_count() >= nproc else "gloo"
    with tempfile.TemporaryDirectory() as td:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
               "--master-addr", "127.0.0.1", "--master-port", str(free_port()),
               os.path.join(ROOT, "tests", "mp_gin_worker.py"), json.dumps(cases), td, transport]
        env = dict(os.environ, OMP_NUM_THREADS="2")
        p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=timeout, text=True)
        if p.returncode != 0 and "Address already in use" in p.stdout:  # lost the race for the rendezvous port
            cmd[cmd.index("--master-port") + 1] = str(free_port())
            p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=timeout, text=True)
        assert p.returncode == 0, "worker failed:\n" + p.stdout[-6000:]
        out = {}
        for c in cases:
            out[c["name"]] = []
            for r in range(nproc):
                z = np.load(os.path.join(td, f"{c['name']}_rank{r}.npz"), allow_pickle=False)
                out[c["name"]].append({k: z[k] for k in z.files})
        return out


def rows_of(d, key, N):
    top, n = (int(x) for x in d[key])
    hi = min(top + n, N)
    return top, hi, hi - top


def close(got, want, tol):
    return np.abs(got - want).max() <= tol * max(np.abs(want).max(), 1.0)


def check_op(c, ranks):
    N, rows, cols = global_graph(c)
    X, dA = global_inputs(c, N)
    f = c["f"]
    E = go.edge_rows(rows, cols, f)
    assert (X[cols] + E == 0).any()
    want = go.edge_relu_aggregate(rows, cols, N, X, E)
    wdX, _ = go.edge_relu_aggregate_backward(rows, cols, X, E, dA, N)
    for r, d in enumerate(ranks):
        top, hi, n = rows_of(d, "topA", N)
        assert close(d["A"][:n], want[top:hi], 1e-13), (c["name"], r)
        assert not d["A"][n:].any()
        top, hi, n = rows_of(d, "topB", N)
        assert close(d["dX"][:n], wdX[top:hi], 1e-12), (c["name"], r)
        ra, ca = d["ra"].astype(np.int64), d["ca"].astype(np.int64)
        _, wdE = go.edge_relu_aggregate_backward(ra, ca, X, go.edge_rows(ra, ca, f), dA, N)
        assert d["dE"].shape == (len(ra), f) and np.array_equal(d["dE"], wdE), (c["name"], r)
        for k in ("A", "dX", "dE"):
            assert np.array_equal(d[k + "2"], d[k]), (c["name"], r, k, "repeat differs")


def attr(c, rows, cols):
    return go.attr_of(rows, cols, c["edge_dim"]) if c["edge_dim"] else None


def check_model(c, ranks):
    N, rows, cols = global_graph(c)
    params, X, G, _ = global_inputs(c, N)
    out, dX, dP = go.forward_backward(rows, cols, N, LAYERS, params, X, G, attr(c, rows, cols))
    for r, d in enumerate(ranks):
        top, hi, n = rows_of(d, "topA", N)
        assert close(d["out"][:n], out[top:hi], 1e-9), (c["name"], r)
        top, hi, n = rows_of(d, "topB", N)
        assert close(d["dX"][:n], dX[top:hi], 1e-9), (c["name"], r)
        for l, grads in enumerate(dP):
            for k, g in grads.items():
                assert np.array_equal(d[f"g{l}_{k}"], ranks[0][f"g{l}_{k}"]), (c["name"], r, l, k, "differs across ranks")
                assert close(d[f"g{l}_{k}"], g, 1e-9), (c["name"], l, k)


def check_train(c, ranks):
    N, rows, cols = global_graph(c)
    params, X, _, labels = global_inputs(c, N)
    res, trained = go.train(rows, cols, N, LAYERS, params, X, labels, 3, attr=attr(c, rows, cols), lr=1e-2, max_grad_norm=0.5)
    for r, d in enumerate(ranks):
        assert np.array_equal(d["steps"], ranks[0]["steps"]), (c["name"], r)
        for t, w in enumerate(res):
            g = d["steps"][t]
            assert abs(g[0] - w[0]) <= 1e-9 * abs(w[0]) and abs(g[3] - w[3]) <= 1e-9 * abs(w[3]), (c["name"], t, g, w)
            assert (int(g[1]), int(g[2])) == (w[1], w[2]), (c["name"], t)
        for l, P in enumerate(trained):
            for k, v in P.items():
                assert np.array_equal(d[f"p{l}_{k}"], ranks[0][f"p{l}_{k}"]), (c["name"], r, l, k)
                assert close(d[f"p{l}_{k}"], v, 1e-9), (c["name"], l, k)


@pytest.mark.parametrize("nproc", [2, 4])
def test_gin_multirank(nproc):
    cases = CASES[nproc]
    got = run(nproc, cases)
    for c in cases:
        ranks = got[c["name"]]
        if c.get("expect"):
            for r, d in enumerate(ranks):
                assert "error" in d and "code -1" in str(d["error"]) and c["expect"] in str(d["error"]), (c["name"], r)
            continue
        for r, d in enumerate(ranks):
            assert "error" not in d, (c["name"], r, str(d.get("error")))
        {"op": check_op, "gin": check_model, "train": check_train}[c["model"]](c, ranks)
