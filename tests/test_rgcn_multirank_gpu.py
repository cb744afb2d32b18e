"""R-GCN and relational aggregation on several ranks on the GPU (tests/mp_rgcn_worker.py), at p = 2 and 4 on the 1.5D
dense shift with replication reuse at c = 1 and 2 and with local kernel fusion at c = 1: the op's A and dX and the
model's output, input gradient and parameter gradients for each aggregator against tests/rgcn_oracle.py on the global
graph, row by row; repeats, parameter gradients and trained parameters bit-identical on every rank; cases on the skewed
graph of tests/skewed_graph.py with relations hashed from (u, v, copy); and HNH_E_INVALID on every rank for the 1.5D
sparse shift, for local kernel fusion at c = 2, and when one rank's S holds a value that is no relation.

Ranks share cuda:0 over the gloo-backed transport unless there is one GPU per rank (then NCCL)."""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from tests import rgcn_oracle as ro
from tests.mp_rgcn_worker import LAYERS, R, global_graph, global_inputs
from tests.mp_util import ROOT, free_port

pytestmark = pytest.mark.gpu

LAYOUTS = [("15d_fusion1", 1), ("15d_fusion1", 2), ("15d_fusion2", 1)]


def case(model, alg, c, logM=7, seed=0xC0FFEE + 251, **kw):
    name = f"{model}_{alg}_c{c}_" + "_".join(f"{k}{v}" for k, v in sorted(kw.items()))
    return dict(name=name, model=model, alg=alg, c=c, logM=logM, seed=seed, **kw)


CASES = {
    p: [case("op", a, c, f=f) for a, c in LAYOUTS for f in (8, 300)]
    + [case("rgcn", a, c, aggr=g, train=1) for a, c in LAYOUTS for g in ro.AGGREGATIONS]
    + [case("op", "15d_fusion1", 2, f=64, skewed=1), case("rgcn", "15d_fusion1", 2, aggr="mean", skewed=1),
       case("rgcn", "15d_fusion2", 1, aggr="sum", skewed=1)]
    + [case("op", "15d_sparse", 1, f=8, expect="not defined"), case("op", "15d_fusion2", 2, f=8, expect="not defined"),
       case("rgcn", "15d_sparse", 1, aggr="mean", expect="not defined"),
       case("rgcn", "15d_fusion2", 2, aggr="sum", expect="not defined"),
       case("rgcn", "15d_fusion1", 2, aggr="mean", bad_rank=p - 1, expect="relations")]
    for p in (2, 4)
}


def run(nproc, cases, timeout=900):
    """Returns {case name: [per-rank dict]}."""
    transport = "nccl" if torch.cuda.device_count() >= nproc else "gloo"
    with tempfile.TemporaryDirectory() as td:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
               "--master-addr", "127.0.0.1", "--master-port", str(free_port()),
               os.path.join(ROOT, "tests", "mp_rgcn_worker.py"), json.dumps(cases), td, transport]
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


def check_op(c, ranks):
    N, rows, cols, rels = global_graph(c)
    X, dA = global_inputs(c, N)
    wA = ro.relational_aggregate(rows, cols, rels, N, X, R)
    wdX = ro.relational_aggregate_backward(rows, cols, rels, dA, N, R)
    for r, d in enumerate(ranks):
        top, hi, n = rows_of(d, "topA", N)
        assert np.abs(d["A"][:n] - wA[top:hi]).max() <= 1e-13 * np.abs(wA).max(), (c["name"], r)
        assert not d["A"][n:].any()
        top, hi, n = rows_of(d, "topB", N)
        assert np.abs(d["dX"][:n] - wdX[top:hi]).max() <= 1e-13 * np.abs(wdX).max(), (c["name"], r)
        assert np.array_equal(d["A2"], d["A"]) and np.array_equal(d["dX2"], d["dX"]), (c["name"], r, "repeat differs")


def check_model(c, ranks):
    N, rows, cols, rels = global_graph(c)
    params, X, G = global_inputs(c, N)
    out, dX, dP = ro.forward_backward(rows, cols, rels, N, LAYERS, params, X, R, c["aggr"], G)
    for r, d in enumerate(ranks):
        top, hi, n = rows_of(d, "topA", N)
        assert np.abs(d["out"][:n] - out[top:hi]).max() <= 1e-10 * np.abs(out).max(), (c["name"], r)
        top, hi, n = rows_of(d, "topB", N)
        assert np.abs(d["dX"][:n] - dX[top:hi]).max() <= 1e-10 * np.abs(dX).max(), (c["name"], r)
        for l, grads in enumerate(dP):
            for k, g in grads.items():
                assert np.array_equal(d[f"g{l}_{k}"], ranks[0][f"g{l}_{k}"]), (c["name"], r, l, k, "differs across ranks")
                assert np.abs(d[f"g{l}_{k}"] - g).max() <= 1e-10 * max(np.abs(g).max(), 1e-300), (c["name"], l, k)
                if c.get("train"):
                    assert np.array_equal(d[f"t{l}_{k}"], ranks[0][f"t{l}_{k}"]), (c["name"], r, l, k, "trained differs")


@pytest.mark.parametrize("nproc", [2, 4])
def test_rgcn_multirank(nproc):
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
        (check_op if c["model"] == "op" else check_model)(c, ranks)
