"""Attention dropout in fused sparse attention on several ranks on the GPU (tests/mp_sparse_attention_dropout_worker.py):
every rank's rows of Z, L, dQ, dK and dV against the global fp64 model on the layouts of
tests/test_sparse_attention_multirank_gpu.py -- the 1.5D dense shift with replication reuse (c = 1, 2) and with local
kernel fusion (c = 1) at p = 2 and 4.  The model keys the mask by global S-row and S-column, so this shows that every
value order, block and ring step of every layout hands the kernels the right offsets.

Ranks share cuda:0 over the gloo-backed transport unless there is one GPU per rank (then NCCL)."""
import json
import math
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from oracle import hnh_oracle as orc
from tests import sparse_attention_dropout_oracle as sd
from tests.mp_sparse_attention_worker import global_inputs
from tests.mp_util import ROOT, free_port
from tests.test_sparse_attention_multirank_gpu import rel_err

pytestmark = pytest.mark.gpu


def case(alg, c, heads=2, d=4, logM=7, npr=5, seed=0xC0FFEE + 33, dropout=0.6, mask_seed=11, **kw):
    return dict(name=f"{alg}_c{c}_h{heads}_p{dropout}", alg=alg, c=c, heads=heads, d=d, logM=logM, npr=npr, seed=seed,
                dropout=dropout, mask_seed=mask_seed, **kw)


CASES = {
    2: [case("15d_fusion1", 1), case("15d_fusion1", 2, heads=1, d=8, dropout=0.1), case("15d_fusion2", 1, heads=4)],
    4: [case("15d_fusion1", 1, heads=1, d=8), case("15d_fusion1", 2, dropout=0.1), case("15d_fusion2", 1, mask_seed=2 ** 64 - 1)],
}


def run(nproc, cases, timeout=900):
    """Returns {case name: [per-rank dict]}."""
    transport = "nccl" if torch.cuda.device_count() >= nproc else "gloo"
    with tempfile.TemporaryDirectory() as td:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
               "--master-addr", "127.0.0.1", "--master-port", str(free_port()),
               os.path.join(ROOT, "tests", "mp_sparse_attention_dropout_worker.py"), json.dumps(cases), td, transport]
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
def test_sparse_attention_dropout_multirank(nproc):
    cases = CASES[nproc]
    got = run(nproc, cases)
    for c in cases:
        N = 1 << c["logM"]
        rows, cols, _ = orc.er_tuples(c["logM"], c["npr"], c["seed"])
        Q, K, V, dZ = global_inputs(N, c["heads"] * c["d"], c["seed"])
        scale = 1 / math.sqrt(c["d"])
        args = (c["heads"], scale, c["dropout"], c["mask_seed"])
        Zw, Lw = sd.forward_np(rows, cols, N, Q, K, V, *args)
        dQw, dKw, dVw = sd.backward_np(rows, cols, N, Q, K, V, dZ, *args)
        coveredA, coveredB = np.zeros(N, bool), np.zeros(N, bool)
        for r, d in enumerate(got[c["name"]]):
            assert "error" not in d, (c["name"], r, str(d.get("error")))
            topA, nrA, topB, nrB = (int(d[k]) for k in ("topA", "nrA", "topB", "nrB"))
            nA, nB = min(nrA, N - topA), min(nrB, N - topB)
            for key, want, top, n in (("Z", Zw, topA, nA), ("L", Lw, topA, nA), ("dQ", dQw, topA, nA),
                                      ("dK", dKw, topB, nB), ("dV", dVw, topB, nB)):
                assert rel_err(d[key][:n], want[top:top + n]) < 1e-10, (c["name"], r, key)
            coveredA[topA:topA + nA] = True
            coveredB[topB:topB + nB] = True
        assert coveredA.all() and coveredB.all(), c["name"]
