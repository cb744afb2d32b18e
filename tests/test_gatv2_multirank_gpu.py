"""GATv2 attention on several ranks on the GPU (tests/mp_gatv2_worker.py): the GATv2 GAT's output rows, input-gradient
rows, weight gradients and attention gradients against the autograd model on the 1.5D dense shift with replication
reuse (c = 1, 2; the stored-row side rides, with its gradient on the backward) and with local kernel fusion (c = 1;
the gathered side rides), the gradients bit-identical on every rank, and the layouts without GATv2 attention
rejected on every rank with HNH_E_INVALID while the workers still exit cleanly.

Ranks share cuda:0 over the gloo-backed transport unless there is one GPU per rank (then NCCL), as in
tests/test_gat_additive_multirank_gpu.py."""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from oracle import hnh_oracle as orc
from tests import gatv2_oracle as g2
from tests.mp_gat_backward_worker import output_grad
from tests.mp_util import ROOT, free_port
from tests.mp_worker import gat_inputs

pytestmark = pytest.mark.gpu

GAT = dict(layers=[[6, 4, 2], [8, 3, 3]], alpha=0.2)


def case(alg, c, logM=7, npr=5, seed=0xC0FFEE + 9, **kw):
    return dict(name=f"{alg}_c{c}", alg=alg, c=c, logM=logM, npr=npr, seed=seed, **{**GAT, **kw})


SUPPORTED = {
    2: [case("15d_fusion1", 1), case("15d_fusion1", 2), case("15d_fusion2", 1)],
    4: [case("15d_fusion1", 1), case("15d_fusion1", 2), case("15d_fusion2", 1)],
}
# (the 1.5D sparse layout splits every width by p / c: even widths)
REJECTED = [case("15d_fusion2", 2, rejected=True), case("15d_sparse", 1, rejected=True, layers=[[6, 4, 2], [8, 2, 2]]),
            case("25d_dense_replicate", 2, rejected=True, layers=[[6, 4, 2], [8, 2, 2]]),
            case("25d_sparse_replicate", 2, rejected=True, layers=[[6, 4, 2], [8, 2, 2]])]


def run(nproc, cases, timeout=900):
    """Returns {case name: [per-rank dict]}."""
    transport = "nccl" if torch.cuda.device_count() >= nproc else "gloo"
    with tempfile.TemporaryDirectory() as td:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
               "--master-addr", "127.0.0.1", "--master-port", str(free_port()),
               os.path.join(ROOT, "tests", "mp_gatv2_worker.py"), json.dumps(cases), td, transport]
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
    return np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-300)


@pytest.mark.parametrize("nproc", [2, 4])
def test_gatv2_multirank(nproc):
    cases = SUPPORTED[nproc]
    got = run(nproc, cases)
    for c in cases:
        N = 1 << c["logM"]
        rows, cols, _ = orc.er_tuples(c["logM"], c["npr"], c["seed"])
        ranks = got[c["name"]]
        layers, X0, weights = gat_inputs(N, c["layers"], c["seed"])
        a = g2.attention_inputs(layers, c["seed"])
        G = output_grad(N, layers[-1][1] * layers[-1][2], c["seed"])
        want_out = g2.gatv2_forward_global(rows, cols, N, layers, weights, a, c["alpha"], X0)
        dX0, dW, da = g2.gatv2_backward_global(rows, cols, N, layers, weights, a, c["alpha"], X0, G)
        covered = np.zeros(N, bool)
        for r, d in enumerate(ranks):
            assert "gat_error" not in d, (c["name"], r, str(d.get("gat_error")))
            topA, nrA, topB, nrB = (int(d[k]) for k in ("topA", "nrA", "topB", "nrB"))
            assert rel_err(d["out"][:nrA], want_out[topA:topA + nrA]) < 1e-10, (c["name"], r)
            assert rel_err(d["dX0"][:nrB], dX0[topB:topB + nrB]) < 1e-10, (c["name"], r)
            covered[topB:topB + nrB] = True
            for i, (_, _, heads) in enumerate(layers):
                for h in range(heads):
                    for key in ("dW", "da"):
                        k = f"{key}_{i}_{h}"
                        assert np.array_equal(d[k], ranks[0][k]), (c["name"], r, k)
        assert covered.all(), c["name"]
        for i, (_, _, heads) in enumerate(layers):
            for h in range(heads):
                for key, want in (("dW", dW), ("da", da)):
                    assert np.abs(want[i][h]).max() > 0, (c["name"], key, i, h)
                    assert rel_err(ranks[0][f"{key}_{i}_{h}"], want[i][h]) < 1e-10, (c["name"], key, i, h)


def test_layouts_without_gatv2_attention_are_rejected_on_every_rank():
    """1.5D dense shift with local kernel fusion at c = 2, the R-split 1.5D sparse shift (c = 1) and both 2.5D
    algorithms (c = 2) at p = 2: gatv2_scores, gatv2_backward and the GATv2 GAT's forward pass raise HNH_E_INVALID naming the configuration
    on every rank, nothing hangs, the workers exit cleanly."""
    got = run(2, REJECTED)
    for c in REJECTED:
        for r, d in enumerate(got[c["name"]]):
            for key, op in (("scores_error", "gatv2Scores"), ("backward_error", "gatv2Backward"),
                            ("gat_error", "GAT GATv2 attention")):
                assert key in d, (c["name"], r, key)
                msg = str(d[key])
                assert "code -1" in msg and op + ": not defined for" in msg and "p = 2" in msg, (c["name"], r, msg)
