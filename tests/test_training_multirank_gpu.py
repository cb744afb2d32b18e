"""Training on several ranks on the GPU (tests/mp_training_worker.py): 3 train steps of the graph transformer (with
blocks, the gate, edge features, dropout and clipping) and of GAT on the 1.5D dense shift with replication reuse (c = 1,
2) and with local kernel fusion (c = 1) at p = 2 and 4.  Loss, correct count, labelled count and gradient norm are equal
on every rank, the trained parameters are bit-identical on every rank and within 1e-9 of tests/training_oracle.py's
global run (the key bias by |delta| <= steps * lr: its gradient is rounding noise).  A layout the model refuses is
refused by train_step on every rank.

Ranks share cuda:0 over the gloo-backed transport unless there is one GPU per rank (then NCCL)."""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from oracle import hnh_oracle as orc
from tests import training_oracle as tro
from tests.mp_graph_transformer_worker import attr_of
from tests.mp_training_worker import global_inputs
from tests.mp_util import ROOT, free_port

pytestmark = pytest.mark.gpu

GT_LAYERS = [[6, 4, 2], [8, 5, 1]]
GAT_LAYERS = [[8, 4, 2], [8, 6, 1]]


def case(model, alg, c, steps=3, logM=7, npr=5, seed=0xC0FFEE + 151, **kw):
    base = dict(layers=GT_LAYERS, edge_dim=3, beta=True, ffn=2, dropout=0.3, clip=0.05) if model == "gt" else \
        dict(layers=GAT_LAYERS, kind="additive", dropout=0.0)
    base.update(kw)
    name = f"{model}_{alg}_c{c}_" + "_".join(f"{k}{v}" for k, v in sorted(kw.items()))
    return dict(name=name, model=model, alg=alg, c=c, steps=steps, logM=logM, npr=npr, seed=seed, **base)


CASES = {
    2: [case("gt", "15d_fusion1", 1), case("gt", "15d_fusion1", 2, ffn=0, edge_dim=0, dropout=0.0),
        case("gt", "15d_fusion2", 1, beta=False), case("gat", "15d_fusion1", 1),
        case("gat", "15d_sparse", 1, kind="leaky", error=True)],
    4: [case("gt", "15d_fusion1", 1, ffn=1, clip=None), case("gt", "15d_fusion1", 2), case("gt", "15d_fusion2", 1, edge_dim=0),
        case("gat", "15d_fusion2", 1, kind="softmax"), case("gat", "15d_fusion2", 2, kind="leaky", error=True),
        case("gat", "25d_dense_replicate", 1, kind="leaky", error=True)],
}


def run(nproc, cases, timeout=900):
    """Returns {case name: [per-rank dict]}."""
    transport = "nccl" if torch.cuda.device_count() >= nproc else "gloo"
    with tempfile.TemporaryDirectory() as td:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
               "--master-addr", "127.0.0.1", "--master-port", str(free_port()),
               os.path.join(ROOT, "tests", "mp_training_worker.py"), json.dumps(cases), td, transport]
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


def oracle(c):
    """(per-step results, {key: trained parameter}) of the global run, keyed as the worker keys them."""
    N, layers = 1 << c["logM"], [tuple(l) for l in c["layers"]]
    rows, cols, _ = orc.er_tuples(c["logM"], c["npr"], c["seed"])
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    params, X, labels = global_inputs(c)
    if c["model"] == "gt":
        res, trained = tro.train_gt(rows, cols, N, layers, params, X, labels, c["steps"],
                                    attr=attr_of(rows, cols, c["edge_dim"]) if c["edge_dim"] else None, beta=c["beta"],
                                    ffn=c["ffn"], dropout=c["dropout"], seeds=[5 + t for t in range(c["steps"])], lr=1e-2,
                                    max_grad_norm=c["clip"])
        return res, {f"p{l}_{k}": v for l, P in enumerate(trained) for k, v in P.items()}
    res, ws, u1, u2 = tro.train_gat(c["kind"], rows, cols, N, layers, *params, X, labels, c["steps"], lr=1e-2)
    want = {}
    for l, (_, _, H) in enumerate(layers):
        for h in range(H):
            want[f"w{l}_{h}"], want[f"a1_{l}_{h}"], want[f"a2_{l}_{h}"] = ws[l][h], u1[l][h], u2[l][h]
    return res, want


@pytest.mark.parametrize("nproc", [2, 4])
def test_training_multirank(nproc):
    cases = CASES[nproc]
    got = run(nproc, cases)
    for c in cases:
        ranks = got[c["name"]]
        if c.get("error"):
            for r, d in enumerate(ranks):
                assert "error" in d and "not defined" in str(d["error"]) and "code -1" in str(d["error"]), (c["name"], r)
            continue
        for r, d in enumerate(ranks):
            assert "error" not in d, (c["name"], r, str(d.get("error")))
            assert np.array_equal(d["steps"], ranks[0]["steps"]), (c["name"], r)
            for k in d:
                assert np.array_equal(d[k], ranks[0][k]), (c["name"], r, k, "differs across ranks")
        res, want = oracle(c)
        steps = ranks[0]["steps"]
        for t, w in enumerate(res):
            assert abs(steps[t][0] - w[0]) <= 1e-10 * abs(w[0]) and abs(steps[t][3] - w[3]) <= 1e-10 * abs(w[3]), (c["name"], t)
            assert (int(steps[t][1]), int(steps[t][2])) == (w[1], w[2]), (c["name"], t)
        for k, w in want.items():
            g = ranks[0][k]
            if k.endswith("_key_bias"):
                assert np.abs(g - w).max() <= c["steps"] * 1e-2 * 1.01, (c["name"], k)
            else:
                assert np.abs(g - w).max() <= 1e-9 * max(np.abs(w).max(), 1.0), (c["name"], k, np.abs(g - w).max())
