"""Graph transformer blocks on several ranks on the GPU (tests/mp_graph_transformer_block_worker.py): every rank's rows
of the output and of the input gradient against the global fp64 model, row by row, and every parameter gradient, the
block's included, against the model's on every rank, bit-identical across ranks; on the 1.5D dense shift with
replication reuse (c = 1, 2) and with local kernel fusion (c = 1) at p = 2 and 4, with edge features, the gate and
dropout.  On layouts where the model is not defined every rank raises HNH_E_INVALID.

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
from tests import graph_transformer_block_oracle as gbo
from tests.mp_graph_transformer_block_worker import global_inputs
from tests.mp_graph_transformer_worker import attr_of
from tests.mp_util import ROOT, free_port
from tests.test_graph_transformer_gpu import grad_err

pytestmark = pytest.mark.gpu

LAYERS = [[6, 4, 2], [8, 3, 3]]


def case(alg, c, ffn=2, edge_dim=3, beta=True, dropout=0.3, logM=7, npr=5, seed=0xC0FFEE + 97, mask_seed=31, **kw):
    return dict(name=f"{alg}_c{c}_f{ffn}_e{edge_dim}_b{int(beta)}_p{dropout}", alg=alg, c=c, layers=LAYERS, ffn=ffn,
                edge_dim=edge_dim, beta=beta, dropout=dropout, logM=logM, npr=npr, seed=seed, mask_seed=mask_seed, **kw)


CASES = {
    2: [case("15d_fusion1", 1), case("15d_fusion1", 2, ffn=1, edge_dim=0, dropout=0.0), case("15d_fusion2", 1, beta=False),
        case("15d_sparse", 1, error=True)],
    4: [case("15d_fusion1", 1, ffn=1, beta=False, dropout=0.0), case("15d_fusion1", 2), case("15d_fusion2", 1, edge_dim=0),
        case("15d_fusion2", 2, error=True), case("15d_sparse", 2, error=True)],
}


def run(nproc, cases, timeout=900):
    """Returns {case name: [per-rank dict]}."""
    transport = "nccl" if torch.cuda.device_count() >= nproc else "gloo"
    with tempfile.TemporaryDirectory() as td:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
               "--master-addr", "127.0.0.1", "--master-port", str(free_port()),
               os.path.join(ROOT, "tests", "mp_graph_transformer_block_worker.py"), json.dumps(cases), td, transport]
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


@pytest.mark.parametrize("nproc", [2, 4])
def test_graph_transformer_block_multirank(nproc):
    cases = CASES[nproc]
    got = run(nproc, cases)
    for c in cases:
        if c.get("error"):
            for r, d in enumerate(got[c["name"]]):
                assert "error" in d and "not defined" in str(d["error"]) and "code -1" in str(d["error"]), (c["name"], r)
            continue
        N = 1 << c["logM"]
        layers = [tuple(l) for l in c["layers"]]
        rows, cols, _ = orc.er_tuples(c["logM"], c["npr"], c["seed"])
        rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
        params, X, G = global_inputs(N, layers, c["edge_dim"], c["beta"], c["ffn"], c["seed"] + 1)
        kw = dict(attr=attr_of(rows, cols, c["edge_dim"]) if c["edge_dim"] else None, beta=c["beta"], p=c["dropout"],
                  seed=c["mask_seed"])
        Yw = gbo.forward_np(rows, cols, N, layers, params, X, **kw)
        dXw, dPw = gbo.backward_np(rows, cols, N, layers, params, X, G, **kw)
        coveredA, coveredB = np.zeros(N, bool), np.zeros(N, bool)
        ranks = got[c["name"]]
        for r, d in enumerate(ranks):
            assert "error" not in d, (c["name"], r, str(d.get("error")))
            topA, nrA, topB, nrB = (int(d[k]) for k in ("topA", "nrA", "topB", "nrB"))
            nA, nB = min(nrA, N - topA), min(nrB, N - topB)
            for key, want, top, n in (("Y", Yw, topA, nA), ("dX", dXw, topB, nB)):
                err = np.abs(d[key][:n] - want[top:top + n]).max(1) / np.abs(want).max()
                assert (err < 1e-10).all(), (c["name"], r, key, int(np.argmax(err)), err.max())
            for l, grads in enumerate(dPw):
                scale = max(np.abs(g).max() for g in grads.values())
                assert set(gbo.BLOCK) <= set(grads)
                for pname, g in grads.items():
                    key = f"g{l}_{pname}"
                    assert grad_err(d[key], g, scale) < 1e-10, (c["name"], r, key)
                    assert np.array_equal(d[key], ranks[0][key]), (c["name"], r, key, "differs across ranks")
            coveredA[topA:topA + nA] = True
            coveredB[topB:topB + nB] = True
        assert coveredA.all() and coveredB.all(), c["name"]
