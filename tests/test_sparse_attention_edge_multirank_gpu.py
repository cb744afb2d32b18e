"""Edge features in fused sparse attention on several ranks on the GPU (tests/mp_sparse_attention_edge_worker.py):
every rank's rows of Z, L, dQ, dK and dV and its dE against the global fp64 model, on the 1.5D dense shift with
replication reuse (c = 1, 2) and with local kernel fusion (c = 1) at p = 2 and 4, with and without a masking bias and
dropout.  Each rank builds its E in both orders from entry_coordinates, and its dE rows are matched to the model's by
(global S-row, S-column), so this shows that every value order, block and ring step hands the kernels the right rows
of E.  On layouts where sparse attention is not defined every rank raises
HNH_E_INVALID.

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
from tests import sparse_attention_edge_oracle as se
from tests.mp_sparse_attention_bias_worker import bias_of
from tests.mp_sparse_attention_edge_worker import edge_of
from tests.mp_sparse_attention_worker import global_inputs
from tests.mp_util import ROOT, free_port
from tests.test_sparse_attention_multirank_gpu import rel_err

pytestmark = pytest.mark.gpu


def case(alg, c, heads=2, d=4, logM=7, npr=5, seed=0xC0FFEE + 53, dropout=0.0, mask_seed=13, bias=False, **kw):
    return dict(name=f"{alg}_c{c}_h{heads}_p{dropout}_b{int(bias)}", alg=alg, c=c, heads=heads, d=d, logM=logM, npr=npr,
                seed=seed, dropout=dropout, mask_seed=mask_seed, bias=bias, **kw)


CASES = {
    2: [case("15d_fusion1", 1), case("15d_fusion1", 2, heads=1, d=8, dropout=0.3), case("15d_fusion2", 1, heads=4, bias=True),
        case("15d_sparse", 1, error=True)],
    4: [case("15d_fusion1", 1, heads=1, d=8, bias=True), case("15d_fusion1", 2, dropout=0.3, bias=True),
        case("15d_fusion2", 1, dropout=0.3), case("15d_fusion2", 2, error=True)],
}


def run(nproc, cases, timeout=900):
    """Returns {case name: [per-rank dict]}."""
    transport = "nccl" if torch.cuda.device_count() >= nproc else "gloo"
    with tempfile.TemporaryDirectory() as td:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
               "--master-addr", "127.0.0.1", "--master-port", str(free_port()),
               os.path.join(ROOT, "tests", "mp_sparse_attention_edge_worker.py"), json.dumps(cases), td, transport]
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


def _lookup(N, rows, cols, values, qr, qc):
    """The per-entry rows of `values` (over the global entries rows, cols) at the entries (qr, qc); stored duplicates
    of one (u, v) carry the same row."""
    key = rows * N + cols
    order = np.argsort(key, kind="stable")
    at = order[np.searchsorted(key[order], qr * N + qc)]
    assert np.array_equal(key[at], qr * N + qc)
    return values[at]


@pytest.mark.parametrize("nproc", [2, 4])
def test_sparse_attention_edge_multirank(nproc):
    cases = CASES[nproc]
    got = run(nproc, cases)
    for c in cases:
        if c.get("error"):
            for r, d in enumerate(got[c["name"]]):
                assert "error" in d and "not defined" in str(d["error"]), (c["name"], r)
            continue
        N = 1 << c["logM"]
        heads = c["heads"]
        rows, cols, _ = orc.er_tuples(c["logM"], c["npr"], c["seed"])
        rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
        Q, K, V, dZ = global_inputs(N, heads * c["d"], c["seed"])
        scale = 1 / math.sqrt(c["d"])
        E = edge_of(rows, cols, heads * c["d"])
        bias = bias_of(rows, cols, 0) if c["bias"] else None
        args = (heads, scale, c["dropout"], c["mask_seed"])
        Zw, Lw = se.forward_np(rows, cols, N, Q, K, V, E, *args, bias=bias)
        dQw, dKw, dVw, dEw, _ = se.backward_np(rows, cols, N, Q, K, V, E, dZ, *args, bias=bias)
        coveredA, coveredB = np.zeros(N, bool), np.zeros(N, bool)
        for r, d in enumerate(got[c["name"]]):
            assert "error" not in d, (c["name"], r, str(d.get("error")))
            topA, nrA, topB, nrB = (int(d[k]) for k in ("topA", "nrA", "topB", "nrB"))
            nA, nB = min(nrA, N - topA), min(nrB, N - topB)
            for key, want, top, n in (("Z", Zw, topA, nA), ("L", Lw, topA, nA), ("dQ", dQw, topA, nA),
                                      ("dK", dKw, topB, nB), ("dV", dVw, topB, nB)):
                assert rel_err(d[key][:n], want[top:top + n]) < 1e-10, (c["name"], r, key)
            want = _lookup(N, rows, cols, dEw, d["rA"], d["cA"])
            assert d["dE"].shape == want.shape, (c["name"], r)
            assert rel_err(d["dE"], want) < 1e-10, (c["name"], r, "dE")
            coveredA[topA:topA + nA] = True
            coveredB[topB:topB + nB] = True
        assert coveredA.all() and coveredB.all(), c["name"]
