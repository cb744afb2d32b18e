"""Additive graph attention on several ranks on the GPU (tests/mp_gat_additive_worker.py): the row and column keys of
both value orders against the coordinates recovered by SDDMMs of index columns, the world row and column sums against
numpy over the global matrix, the additive GAT's output rows, input-gradient rows, weight gradients and attention
gradients against the autograd model, the gradients bit-identical on every rank, and the layouts without additive
attention rejected on every rank with HNH_E_INVALID while the workers still exit cleanly.

Ranks share cuda:0 over the gloo-backed transport unless there is one GPU per rank (then NCCL), as in
tests/test_edge_softmax_multirank_gpu.py."""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from oracle import hnh_oracle as orc
from tests import gat_additive_oracle as gao
from tests.mp_gat_additive_worker import summand
from tests.mp_gat_backward_worker import output_grad
from tests.mp_util import ROOT, free_port
from tests.mp_worker import gat_inputs

pytestmark = pytest.mark.gpu

GAT = dict(layers=[[6, 4, 2], [8, 3, 3]], alpha=0.2)


def case(alg, c, logM=7, npr=5, seed=0xC0FFEE + 6, **kw):
    return dict(name=f"{alg}_c{c}", alg=alg, c=c, logM=logM, npr=npr, seed=seed, **{**GAT, **kw})


SUPPORTED = {
    2: [case("15d_fusion1", 1), case("15d_fusion1", 2), case("15d_fusion2", 1)],
    4: [case("15d_fusion1", 1), case("15d_fusion1", 2), case("15d_fusion2", 1)],
}
# (the 1.5D sparse layout splits every width by p / c: even widths)
REJECTED = [case("15d_fusion2", 2, rejected=True), case("15d_sparse", 1, rejected=True, layers=[[6, 4, 2], [8, 2, 2]])]


def run(nproc, cases, timeout=900):
    """Returns {case name: [per-rank dict]}."""
    transport = "nccl" if torch.cuda.device_count() >= nproc else "gloo"
    with tempfile.TemporaryDirectory() as td:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
               "--master-addr", "127.0.0.1", "--master-port", str(free_port()),
               os.path.join(ROOT, "tests", "mp_gat_additive_worker.py"), json.dumps(cases), td, transport]
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
def test_additive_gat_multirank(nproc):
    cases = SUPPORTED[nproc]
    got = run(nproc, cases)
    for c in cases:
        N = 1 << c["logM"]
        rows, cols, _ = orc.er_tuples(c["logM"], c["npr"], c["seed"])
        ri, ci = (t.numpy() for t in gao.edges(rows, cols, N))
        ranks = got[c["name"]]
        # keys: every stored entry appears once over the ranks in each order, with its own row and column
        for mode in ("A", "B"):
            at = []
            for r, d in enumerate(ranks):
                assert "keys_error" not in d, (c["name"], r, str(d.get("keys_error")))
                assert np.array_equal(d[f"{mode}_row_keys"], d[f"{mode}_rows"]), (c["name"], mode, r)
                assert np.array_equal(d[f"{mode}_col_keys"], d[f"{mode}_cols"]), (c["name"], mode, r)
                at.append(np.searchsorted(ri * N + ci, d[f"{mode}_rows"] * N + d[f"{mode}_cols"]))
            assert np.array_equal(np.sort(np.concatenate(at)), np.arange(len(ri))), (c["name"], mode)
        # world row and column sums: the global sums, identical on every rank
        v = summand(ri, ci)
        for r, d in enumerate(ranks):
            assert rel_err(d["row_sums"], np.bincount(ri, weights=v, minlength=N)) < 1e-13, (c["name"], r)
            assert rel_err(d["col_sums"], np.bincount(ci, weights=v, minlength=N)) < 1e-13, (c["name"], r)
            assert np.array_equal(d["row_sums"], ranks[0]["row_sums"]) and np.array_equal(d["col_sums"], ranks[0]["col_sums"])
        # additive GAT
        layers, X0, weights = gat_inputs(N, c["layers"], c["seed"])
        a1, a2 = gao.attention_inputs(layers, c["seed"])
        G = output_grad(N, layers[-1][1] * layers[-1][2], c["seed"])
        want_out = gao.gat_additive_forward_global(rows, cols, N, layers, weights, a1, a2, c["alpha"], X0)
        dX0, dW, da1, da2 = gao.gat_additive_backward_global(rows, cols, N, layers, weights, a1, a2, c["alpha"], X0, G)
        covered = np.zeros(N, bool)
        for r, d in enumerate(ranks):
            assert "gat_error" not in d, (c["name"], r, str(d.get("gat_error")))
            topA, nrA, topB, nrB = (int(d[k]) for k in ("topA", "nrA", "topB", "nrB"))
            assert rel_err(d["out"][:nrA], want_out[topA:topA + nrA]) < 1e-10, (c["name"], r)
            assert rel_err(d["dX0"][:nrB], dX0[topB:topB + nrB]) < 1e-10, (c["name"], r)
            covered[topB:topB + nrB] = True
            for i, (_, _, heads) in enumerate(layers):
                for h in range(heads):
                    for key in ("dW", "da1", "da2"):
                        k = f"{key}_{i}_{h}"
                        assert np.array_equal(d[k], ranks[0][k]), (c["name"], r, k)
        assert covered.all(), c["name"]
        for i, (_, _, heads) in enumerate(layers):
            for h in range(heads):
                for key, want in (("dW", dW), ("da1", da1), ("da2", da2)):
                    assert np.abs(want[i][h]).max() > 0, (c["name"], key, i, h)
                    assert rel_err(ranks[0][f"{key}_{i}_{h}"], want[i][h]) < 1e-10, (c["name"], key, i, h)


def test_layouts_without_additive_attention_are_rejected_on_every_rank():
    """1.5D dense shift with local kernel fusion at c = 2, and the R-split 1.5D sparse shift at p = 2: additive_scores,
    edge_sums and the additive GAT's forward pass raise HNH_E_INVALID naming the configuration on every rank, nothing
    hangs, the workers exit cleanly."""
    got = run(2, REJECTED)
    for c in REJECTED:
        for r, d in enumerate(got[c["name"]]):
            for key, op in (("scores_error", "additiveScores"), ("sums_error", "edgeSums"),
                            ("gat_error", "GAT additive attention")):
                assert key in d, (c["name"], r, key)
                msg = str(d[key])
                assert "code -1" in msg and op + ": not defined for" in msg and "p = 2" in msg, (c["name"], r, msg)
