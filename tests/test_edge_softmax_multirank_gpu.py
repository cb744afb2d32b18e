"""Edge softmax and softmax graph attention on several ranks on the GPU (tests/mp_edge_softmax_worker.py): both value
orders of edge_softmax / edge_softmax_backward per S row against numpy over the global matrix, the softmax GAT's
output rows, input-gradient rows and weight gradients against the autograd model, the weight gradients
bit-identical on every rank, and the layouts without a row softmax rejected on every rank with HNH_E_INVALID while
the workers still exit cleanly.

Ranks share cuda:0 over the gloo-backed transport unless there is one GPU per rank (then NCCL), as in
tests/test_gat_backward_multirank_gpu.py."""
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
from tests import gat_softmax_oracle as gso
from tests.mp_edge_softmax_worker import masked, score, upstream
from tests.mp_gat_backward_worker import output_grad
from tests.mp_util import ROOT, free_port
from tests.mp_worker import gat_inputs

pytestmark = pytest.mark.gpu

GAT = dict(layers=[[6, 4, 2], [8, 3, 3]], alpha=0.2)


def case(alg, c, logM=7, npr=5, seed=0xC0FFEE + 2, **kw):
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
               os.path.join(ROOT, "tests", "mp_edge_softmax_worker.py"), json.dumps(cases), td, transport]
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
def test_edge_softmax_and_softmax_gat_multirank(nproc):
    cases = SUPPORTED[nproc]
    got = run(nproc, cases)
    for c in cases:
        N = 1 << c["logM"]
        rows, cols, _ = orc.er_tuples(c["logM"], c["npr"], c["seed"])
        ri, ci = (t.numpy() for t in gbo.edges(rows, cols, N))
        ranks = got[c["name"]]
        # edge softmax: every stored entry appears once over the ranks, in each order
        alpha = gso.edge_softmax_np(score(ri, ci), ri, N)
        dx = gso.edge_softmax_backward_np(alpha, upstream(ri, ci), ri, N)
        for mode in ("A", "B"):
            keys = []
            for r, d in enumerate(ranks):
                assert "softmax_error" not in d, (c["name"], r, str(d.get("softmax_error")))
                at = np.searchsorted(ri * N + ci, d[f"{mode}_rows"] * N + d[f"{mode}_cols"])
                assert rel_err(d[f"{mode}_alpha"], alpha[at]) < 1e-13, (c["name"], mode, r)
                assert rel_err(d[f"{mode}_dx"], dx[at]) < 1e-13, (c["name"], mode, r)
                keys.append(at)
            keys = np.concatenate(keys)
            assert np.array_equal(np.sort(keys), np.arange(len(ri))), (c["name"], mode)
        # softmax GAT
        layers, X0, weights = gat_inputs(N, c["layers"], c["seed"])
        G = output_grad(N, layers[-1][1] * layers[-1][2], c["seed"])
        want_out = gso.gat_softmax_forward_global(rows, cols, N, layers, weights, c["alpha"], X0)
        dX0, dW = gso.gat_softmax_backward_global(rows, cols, N, layers, weights, c["alpha"], X0, G)
        covered = np.zeros(N, bool)
        for r, d in enumerate(ranks):
            assert "gat_error" not in d, (c["name"], r, str(d.get("gat_error")))
            topA, nrA, topB, nrB = (int(d[k]) for k in ("topA", "nrA", "topB", "nrB"))
            assert rel_err(d["out"][:nrA], want_out[topA:topA + nrA]) < 1e-10, (c["name"], r)
            assert rel_err(d["dX0"][:nrB], dX0[topB:topB + nrB]) < 1e-10, (c["name"], r)
            covered[topB:topB + nrB] = True
            for i, (_, _, heads) in enumerate(layers):
                for h in range(heads):
                    assert np.array_equal(d[f"dW_{i}_{h}"], ranks[0][f"dW_{i}_{h}"]), (c["name"], r, i, h)
        assert covered.all(), c["name"]
        for i, (_, _, heads) in enumerate(layers):
            for h in range(heads):
                assert rel_err(ranks[0][f"dW_{i}_{h}"], dW[i][h]) < 1e-10, (c["name"], i, h)


def test_layouts_without_a_row_softmax_are_rejected_on_every_rank():
    """1.5D dense shift with local kernel fusion at c = 2, and the R-split 1.5D sparse shift at p = 2: edge_softmax
    and the softmax GAT's forward pass raise HNH_E_INVALID naming the configuration on every rank, nothing hangs,
    the workers exit cleanly."""
    got = run(2, REJECTED)
    for c in REJECTED:
        for r, d in enumerate(got[c["name"]]):
            for key, op in (("softmax_error", "edgeSoftmax"), ("gat_error", "GAT softmax attention")):
                assert key in d, (c["name"], r, key)
                msg = str(d[key])
                assert "code -1" in msg and op + ": not defined for" in msg and "p = 2" in msg, (c["name"], r, msg)


def test_edge_softmax_masked_multirank():
    """-inf scores at p = 2 on rows of about 70 entries: every entry of some rows in the first half of the columns, so
    that a rank whose entries of a row are all masked has a local row maximum of -inf and its share of the row sum must
    rescale to 0, not NaN; and every other entry of other rows, so that -inf is the first entry some lanes see."""
    c = dict(case("15d_fusion1", 1, npr=100), name="15d_fusion1_c1_masked", mask=True)
    ranks = run(2, [c])[c["name"]]
    N = 1 << c["logM"]
    rows, cols, _ = orc.er_tuples(c["logM"], c["npr"], c["seed"])
    ri, ci = (t.numpy() for t in gbo.edges(rows, cols, N))
    x = score(ri, ci)
    x[masked(ri, ci, N)] = -np.inf
    alpha = gso.edge_softmax_np(x, ri, N)  # NaN on the rows masked throughout, as torch.softmax
    dx = gso.edge_softmax_backward_np(alpha, upstream(ri, ci), ri, N)
    finite_rows = np.unique(ri[np.isfinite(x)])
    local_masked = 0
    for mode in ("A", "B"):
        for r, d in enumerate(ranks):
            assert "softmax_error" not in d, (r, str(d.get("softmax_error")))
            at = np.searchsorted(ri * N + ci, d[f"{mode}_rows"] * N + d[f"{mode}_cols"])
            for got, want in ((d[f"{mode}_alpha"], alpha[at]), (d[f"{mode}_dx"], dx[at])):
                nan = np.isnan(want)
                assert np.array_equal(np.isnan(got), nan), (mode, r)
                assert rel_err(got[~nan], want[~nan]) < 1e-13, (mode, r)
            assert np.all(d[f"{mode}_alpha"][np.isneginf(x[at]) & np.isin(d[f"{mode}_rows"], finite_rows)] == 0), (mode, r)
            # rows this rank holds only masked entries of, while another rank holds finite ones
            mine = np.unique(d[f"{mode}_rows"])
            live = np.unique(d[f"{mode}_rows"][np.isfinite(x[at])])
            local_masked += len(np.intersect1d(np.setdiff1d(mine, live), finite_rows))
    assert local_masked > 0
