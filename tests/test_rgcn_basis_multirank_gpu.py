"""R-GCN with basis decomposition on several ranks on the GPU (tests/mp_rgcn_basis_worker.py), at p = 2 and 4 on the 1.5D
dense shift with replication reuse at c = 1 and 2 and with local kernel fusion at c = 1: the op's H, dX and dcomp (with
the mean's scale) and the model's output, input gradient and parameter gradients (comp included) for each aggregator
against tests/rgcn_basis_oracle.py on the global graph, row by row; repeats, dcomp, parameter gradients and trained
parameters bit-identical on every rank; cases on the skewed graph of tests/skewed_graph.py; and HNH_E_INVALID on every
rank for the 1.5D sparse shift and for local kernel fusion at c = 2.

Ranks share cuda:0 over the gloo-backed transport unless there is one GPU per rank (then NCCL)."""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from tests import rgcn_basis_oracle as bo
from tests.mp_rgcn_basis_worker import LAYERS, B, R, global_graph, global_inputs
from tests.mp_util import ROOT, free_port
from tests.test_rgcn_multirank_gpu import rows_of

pytestmark = pytest.mark.gpu

LAYOUTS = [("15d_fusion1", 1), ("15d_fusion1", 2), ("15d_fusion2", 1)]


def case(model, alg, c, logM=7, seed=0xC0FFEE + 269, **kw):
    name = f"{model}_{alg}_c{c}_" + "_".join(f"{k}{v}" for k, v in sorted(kw.items()))
    return dict(name=name, model=model, alg=alg, c=c, logM=logM, seed=seed, **kw)


CASES = ([case("op", a, c, f=f) for a, c in LAYOUTS for f in (8, 300)]
         + [case("rgcn", a, c, aggr=g) for a, c in LAYOUTS for g in bo.AGGREGATIONS]
         + [case("op", "15d_fusion1", 2, f=64, skewed=1), case("rgcn", "15d_fusion1", 2, aggr="mean", skewed=1),
            case("rgcn", "15d_fusion2", 1, aggr="sum", skewed=1)]
         + [case("op", "15d_sparse", 1, f=8, expect="not defined"), case("op", "15d_fusion2", 2, f=8, expect="not defined"),
            case("rgcn", "15d_sparse", 1, aggr="mean", expect="not defined"),
            case("rgcn", "15d_fusion2", 2, aggr="sum", expect="not defined")])


def run(nproc, cases, timeout=900):
    """Returns {case name: [per-rank dict]}."""
    transport = "nccl" if torch.cuda.device_count() >= nproc else "gloo"
    with tempfile.TemporaryDirectory() as td:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
               "--master-addr", "127.0.0.1", "--master-port", str(free_port()),
               os.path.join(ROOT, "tests", "mp_rgcn_basis_worker.py"), json.dumps(cases), td, transport]
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


def check_op(c, ranks):
    N, rows, cols, rels = global_graph(c)
    X, dH, comp = global_inputs(c, N)
    scale = bo.mean_scale(rows, rels, N, R)
    wH = bo.basis_aggregate(rows, cols, rels, N, X, R, comp, scale)
    wdX, wdcomp = bo.basis_aggregate_backward(rows, cols, rels, dH, X, N, R, comp, scale)
    for r, d in enumerate(ranks):
        top, hi, n = rows_of(d, "topA", N)
        assert np.abs(d["H"][:n] - wH[top:hi]).max() <= 1e-12 * np.abs(wH).max(), (c["name"], r)
        assert not d["H"][n:].any()
        top, hi, n = rows_of(d, "topB", N)
        assert np.abs(d["dX"][:n] - wdX[top:hi]).max() <= 1e-12 * np.abs(wdX).max(), (c["name"], r)
        assert np.abs(d["dcomp"] - wdcomp).max() <= 1e-12 * np.abs(wdcomp).max(), (c["name"], r)
        assert np.array_equal(d["dcomp"], ranks[0]["dcomp"]), (c["name"], r, "dcomp differs across ranks")
        for k in ("H", "dX", "dcomp"):
            assert np.array_equal(d[k + "2"], d[k]), (c["name"], r, k, "repeat differs")


def check_model(c, ranks):
    N, rows, cols, rels = global_graph(c)
    params, X, G = global_inputs(c, N)
    out, dX, dP = bo.forward_backward(rows, cols, rels, N, LAYERS, params, X, R, B, c["aggr"], G)
    for r, d in enumerate(ranks):
        top, hi, n = rows_of(d, "topA", N)
        assert np.abs(d["out"][:n] - out[top:hi]).max() <= 1e-10 * np.abs(out).max(), (c["name"], r)
        top, hi, n = rows_of(d, "topB", N)
        assert np.abs(d["dX"][:n] - dX[top:hi]).max() <= 1e-10 * np.abs(dX).max(), (c["name"], r)
        for l, grads in enumerate(dP):
            for k, g in grads.items():
                assert np.array_equal(d[f"g{l}_{k}"], ranks[0][f"g{l}_{k}"]), (c["name"], r, l, k, "differs across ranks")
                assert np.abs(d[f"g{l}_{k}"] - g).max() <= 1e-10 * max(np.abs(g).max(), 1e-300), (c["name"], l, k)
                assert np.array_equal(d[f"t{l}_{k}"], ranks[0][f"t{l}_{k}"]), (c["name"], r, l, k, "trained differs")


@pytest.mark.parametrize("nproc", [2, 4])
def test_rgcn_basis_multirank(nproc):
    got = run(nproc, CASES)
    for c in CASES:
        ranks = got[c["name"]]
        if c.get("expect"):
            for r, d in enumerate(ranks):
                assert "error" in d and "code -1" in str(d["error"]) and c["expect"] in str(d["error"]), (c["name"], r)
            continue
        for r, d in enumerate(ranks):
            assert "error" not in d, (c["name"], r, str(d.get("error")))
        (check_op if c["model"] == "op" else check_model)(c, ranks)
