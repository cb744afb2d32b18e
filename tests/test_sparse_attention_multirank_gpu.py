"""Fused sparse attention on several ranks on the GPU (tests/mp_sparse_attention_worker.py): every rank's rows of Z, L,
dQ, dK and dV against the fp64 model on the 1.5D dense shift with replication reuse (c = 1, 2: the stored-row side rides
with what it accumulates) and with local kernel fusion (c = 1: the gathered side rides), and the layouts without sparse
attention rejected on every rank with HNH_E_INVALID while the workers still exit cleanly.

Ranks share cuda:0 over the gloo-backed transport unless there is one GPU per rank (then NCCL), as in
tests/test_gatv2_multirank_gpu.py."""
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
from tests import sparse_attention_oracle as sa
from tests.mp_sparse_attention_worker import global_inputs
from tests.mp_util import ROOT, free_port

pytestmark = pytest.mark.gpu


def case(alg, c, heads=2, d=4, logM=7, npr=5, seed=0xC0FFEE + 23, **kw):
    return dict(name=f"{alg}_c{c}_h{heads}", alg=alg, c=c, heads=heads, d=d, logM=logM, npr=npr, seed=seed, **kw)


SUPPORTED = {
    2: [case("15d_fusion1", 1), case("15d_fusion1", 2, heads=1, d=8), case("15d_fusion2", 1, heads=4)],
    4: [case("15d_fusion1", 1, heads=1, d=8), case("15d_fusion1", 2), case("15d_fusion2", 1)],
}
# at p = 4 (the 1.5D sparse shift and both 2.5D layouts split the width by c: even head widths)
REJECTED = [case("15d_fusion2", 2, rejected=True), case("15d_sparse", 1, rejected=True),
            case("25d_dense_replicate", 1, rejected=True), case("25d_sparse_replicate", 1, rejected=True)]


def run(nproc, cases, timeout=900):
    """Returns {case name: [per-rank dict]}."""
    transport = "nccl" if torch.cuda.device_count() >= nproc else "gloo"
    with tempfile.TemporaryDirectory() as td:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
               "--master-addr", "127.0.0.1", "--master-port", str(free_port()),
               os.path.join(ROOT, "tests", "mp_sparse_attention_worker.py"), json.dumps(cases), td, transport]
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


def rel_err(got, ref):
    fin = np.isfinite(ref)
    assert np.array_equal(fin, np.isfinite(got)) and np.array_equal(got[~fin], ref[~fin])
    return np.abs(got[fin] - ref[fin]).max(initial=0.0) / max(np.abs(ref[fin]).max(initial=0.0), 1e-300)


@pytest.mark.parametrize("nproc", [2, 4])
def test_sparse_attention_multirank(nproc):
    cases = SUPPORTED[nproc]
    got = run(nproc, cases)
    for c in cases:
        N = 1 << c["logM"]
        rows, cols, _ = orc.er_tuples(c["logM"], c["npr"], c["seed"])
        Q, K, V, dZ = global_inputs(N, c["heads"] * c["d"], c["seed"])
        scale = 1 / math.sqrt(c["d"])
        Zw, Lw = sa.forward_np(rows, cols, N, Q, K, V, c["heads"], scale)
        dQw, dKw, dVw = sa.backward_np(rows, cols, N, Q, K, V, dZ, c["heads"], scale)
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


def test_layouts_without_sparse_attention_are_rejected_on_every_rank():
    """1.5D dense shift with local kernel fusion at c = 2, the R-split 1.5D sparse shift and both 2.5D algorithms at
    p = 4: sparse_attention and sparse_attention_backward raise HNH_E_INVALID naming the configuration on every rank,
    nothing hangs, the workers exit cleanly."""
    got = run(4, REJECTED)
    for c in REJECTED:
        for r, d in enumerate(got[c["name"]]):
            for key, op in (("forward_error", "sparseAttention"), ("backward_error", "sparseAttentionBackward")):
                assert key in d, (c["name"], r, key)
                msg = str(d[key])
                assert "code -1" in msg and op + ": not defined for" in msg and "p = 4" in msg, (c["name"], r, msg)
