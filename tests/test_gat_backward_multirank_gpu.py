"""GAT backward pass on several ranks on the GPU (tests/mp_gat_backward_worker.py): every rank's input-gradient rows
and the weight gradients against the autograd model, the weight gradients bit-identical on every rank, and the
layouts without a backward pass rejected on every rank with HNH_E_INVALID while the workers still exit cleanly.

Ranks share cuda:0 over the gloo-backed transport unless there is one GPU per rank (then NCCL), as in
tests/test_multirank_gpu.py."""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from oracle import hnh_oracle as orc
from tests import gat_backward_oracle as gbo
from tests.mp_gat_backward_worker import output_grad
from tests.mp_util import ROOT, free_port
from tests.mp_worker import gat_inputs

pytestmark = pytest.mark.gpu

GAT = dict(layers=[[6, 4, 2], [8, 3, 3]], alpha=0.2)


def case(alg, c, logM=7, npr=5, seed=0xC0FFEE + 1, **kw):
    return dict(name=f"{alg}_c{c}", alg=alg, c=c, logM=logM, npr=npr, seed=seed, **{**GAT, **kw})


SUPPORTED = {
    2: [case("15d_fusion1", 1), case("15d_fusion2", 1)],
    4: [case("15d_fusion1", 2), case("15d_fusion2", 1)],
    8: [case("15d_fusion1", 2), case("15d_fusion2", 1)],
}
# (the 1.5D sparse layout splits every width by p / c: even widths; its forward pass is not the GAT formula, so the
# backward is called without one -- it must reject the layout first)
REJECTED = {2: [case("15d_fusion2", 2), case("15d_sparse", 1, forward=False, layers=[[6, 4, 2], [8, 2, 2]])]}


def transport_for(nproc):
    return "nccl" if torch.cuda.device_count() >= nproc else "gloo"


def run(nproc, cases, timeout=900):
    """Returns {case name: [per-rank dict]}."""
    with tempfile.TemporaryDirectory() as td:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
               "--master-addr", "127.0.0.1", "--master-port", str(free_port()),
               os.path.join(ROOT, "tests", "mp_gat_backward_worker.py"), json.dumps(cases), td, transport_for(nproc)]
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


@pytest.mark.parametrize("nproc", [2, 4, 8])
def test_gat_backward_multirank_matches_autograd(nproc):
    if nproc == 8 and torch.cuda.device_count() < 8:
        pytest.skip("p = 8 runs where eight GPUs exist")
    cases = SUPPORTED[nproc]
    got = run(nproc, cases)
    for c in cases:
        N = 1 << c["logM"]
        rows, cols, _ = orc.er_tuples(c["logM"], c["npr"], c["seed"])
        layers, X0, weights = gat_inputs(N, c["layers"], c["seed"])
        G = output_grad(N, layers[-1][1] * layers[-1][2], c["seed"])
        dX0, dW = gbo.gat_backward_global(rows, cols, N, layers, weights, c["alpha"], X0, G)
        ranks = got[c["name"]]
        covered = np.zeros(N, bool)
        for r, d in enumerate(ranks):
            assert "error" not in d, (c["name"], r, str(d.get("error")))
            top, nr = int(d["topB"]), int(d["nrB"])
            assert rel_err(d["dX0"][:nr], dX0[top:top + nr]) < 1e-10, (c["name"], r)
            covered[top:top + nr] = True
            for i, (_, _, heads) in enumerate(layers):
                for h in range(heads):
                    # the all-reduced weight gradient is the same on every rank, bit for bit
                    assert np.array_equal(d[f"dW_{i}_{h}"], ranks[0][f"dW_{i}_{h}"]), (c["name"], r, i, h)
        assert covered.all(), c["name"]
        for i, (_, _, heads) in enumerate(layers):
            for h in range(heads):
                assert rel_err(ranks[0][f"dW_{i}_{h}"], dW[i][h]) < 1e-10, (c["name"], i, h)


def test_gat_backward_rejects_layouts_without_one_on_every_rank():
    """1.5D dense shift with local kernel fusion at c = 2, and the R-split 1.5D sparse shift at p = 2: every rank
    gets HNH_E_INVALID naming the configuration, nothing hangs, the workers exit cleanly."""
    got = run(2, REJECTED[2])
    for c in REJECTED[2]:
        for r, d in enumerate(got[c["name"]]):
            assert "error" in d, (c["name"], r)
            msg = str(d["error"])
            assert "code -1" in msg and "not defined for" in msg and "p = 2" in msg, (c["name"], r, msg)
