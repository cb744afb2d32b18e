"""The graph readout on several ranks on the GPU (tests/mp_graph_readout_worker.py), on the 1.5D dense shift with
replication reuse at c = 1 and 2 and with local kernel fusion at c = 1, at p = 2 and 4.  Graphs straddle rank
boundaries, one case leaves a rank without graph rows, and a graph's maximum is attained on two ranks.  The op (sum,
mean, max; pool and pool_backward) against tests/graph_readout_oracle.py, with P bit-identical on every rank and on a
repeat; 3 graph train steps of GraphSAGE (each pool, with and without the head) and of the graph transformer with
dropout, with the steps, the head's parameters and gradients, the model's parameters and the logits bit-identical on
every rank and within 1e-9 of the oracle's global run; and refusals on every rank (a layout without full rows, a bad
batch, another graph count or other labels on one rank only).

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
from tests import graph_readout_oracle as gro
from tests import graph_sage_oracle as gso
from tests import graph_transformer_oracle as gto
from tests.mp_graph_readout_worker import GT_LAYERS, SAGE_LAYERS, global_inputs
from tests.mp_util import ROOT, free_port

pytestmark = pytest.mark.gpu


def case(p, model, alg, c, pool="mean", head=True, steps=3, logM=7, seed=0xC0FFEE + 411, **kw):
    base = dict(r=16, dropout=0.2 if model == "gt" else 0.0, aggr="mean")
    base.update(kw)
    name = f"{model}_{alg}_c{c}_{pool}_h{int(head)}_" + "_".join(f"{k}{v}" for k, v in sorted(kw.items()))
    return dict(name=name, p=p, model=model, alg=alg, c=c, pool=pool, head=head, steps=steps, logM=logM, seed=seed, **base)


LAYOUTS = [("15d_fusion1", 1), ("15d_fusion1", 2), ("15d_fusion2", 1)]
CASES = {
    p: [case(p, "op", a, c, pool, head=False) for a, c in LAYOUTS for pool in gro.POOLS]
    + [case(p, "op", "15d_fusion1", 1, "max", head=False, r=7), case(p, "op", "15d_fusion1", 1, "max", head=False, empty_rank=1)]
    + [case(p, "sage", a, c, "max") for a, c in LAYOUTS]
    + [case(p, "sage", "15d_fusion1", 1, "sum", head=False), case(p, "sage", "15d_fusion2", 1, "mean", aggr="max"),
       case(p, "sage", "15d_fusion1", 2, "sum", empty_rank=p - 1)]
    + [case(p, "gt", a, c, "mean") for a, c in LAYOUTS]
    + [case(p, "gat", "15d_sparse", 1, expect="not defined"), case(p, "gat", "15d_fusion2", 2, expect="not defined"),
       case(p, "sage", "15d_fusion1", 1, bad_batch_rank=p - 1, expect="not below"),
       case(p, "sage", "15d_fusion1", 1, bad_g_rank=p - 1, expect="graph count differs"),
       case(p, "sage", "15d_fusion1", 1, bad_labels_rank=p - 1, expect="labels differ")]
    for p in (2, 4)
}


def run(nproc, cases, timeout=900):
    """Returns {case name: [per-rank dict]}."""
    transport = "nccl" if torch.cuda.device_count() >= nproc else "gloo"
    with tempfile.TemporaryDirectory() as td:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
               "--master-addr", "127.0.0.1", "--master-port", str(free_port()),
               os.path.join(ROOT, "tests", "mp_graph_readout_worker.py"), json.dumps(cases), td, transport]
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


def _close(got, want, tol):
    return np.abs(got - want).max() <= tol * max(np.abs(want).max(), 1.0)


def check_op(c, ranks):
    N = 1 << c["logM"]
    batch, G, _, H, _, _, _ = global_inputs(c)
    h = N // 2
    owner = lambda u: next(r for r, d in enumerate(ranks) if d["top"][0] <= u < d["top"][0] + d["top"][1])  # noqa: E731
    if c.get("empty_rank") is None and c["pool"] == "max":  # the maximum of the straddling graph lies on two ranks
        assert owner(h - 2) != owner(h + 1)
    Ht = torch.from_numpy(H).requires_grad_()
    P = gro.pool_torch(Ht, batch, G, c["pool"])
    dP = np.random.default_rng(c["seed"] + 9).standard_normal((G, H.shape[1]))
    P.backward(torch.from_numpy(dP))
    for r, d in enumerate(ranks):
        assert np.array_equal(d["P"], ranks[0]["P"]) and np.array_equal(d["again"], d["P"]), (c["name"], r)
        top, rows = (int(x) for x in d["top"])
        hi = min(top + rows, N)
        assert _close(d["dH"][:hi - top], Ht.grad.numpy()[top:hi], 1e-12) and not d["dH"][hi - top:].any(), (c["name"], r)
    assert _close(ranks[0]["P"], P.detach().numpy(), 1e-12), c["name"]


def oracle(c):
    N = 1 << c["logM"]
    rows, cols, _ = orc.er_tuples(c["logM"], 5, c["seed"])
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    batch, G, labels, _, params, head, X = global_inputs(c)
    tp = [{k: gso._t(v).clone().requires_grad_() for k, v in P.items()} for P in params]
    x = gso._t(X)
    if c["model"] == "gt":
        fwd = lambda t: gto.model_torch(rows, cols, N, GT_LAYERS, tp, x, None, False, c["dropout"], 5 + t)  # noqa: E731
        evalf = lambda: gto.model_torch(rows, cols, N, GT_LAYERS, tp, x)  # noqa: E731
    else:
        fwd = lambda t: gso.model_torch(rows, cols, N, SAGE_LAYERS, tp, x, c["aggr"])  # noqa: E731
        evalf = lambda: fwd(0)  # noqa: E731
    res, trained_head = gro.train(fwd, [v for P in tp for v in P.values()], batch, G, c["pool"], head, labels, c["steps"], lr=1e-2,
                                  max_grad_norm=0.5)
    with torch.no_grad():
        hl = None if head is None else tuple(gso._t(v) for v in trained_head)
        logits = gro.head_torch(gro.pool_torch(evalf(), batch, G, c["pool"]), hl).numpy()
    want = {f"p{l}_{k}": v.detach().numpy() for l, P in enumerate(tp) for k, v in P.items()}
    if head is not None:
        want["head_weight"], want["head_bias"] = trained_head
    return res, want, logits


@pytest.mark.parametrize("nproc", [2, 4])
def test_graph_readout_multirank(nproc):
    cases = CASES[nproc]
    got = run(nproc, cases)
    for c in cases:
        ranks = got[c["name"]]
        if c.get("expect"):
            for r, d in enumerate(ranks):
                assert "error" in d and "code -1" in str(d["error"]), (c["name"], r, {k: v for k, v in d.items() if k == "error"})
                msg = str(d["error"])
                assert c["expect"] in msg or "another rank" in msg, (c["name"], r, msg)
            continue
        for r, d in enumerate(ranks):
            assert "error" not in d, (c["name"], r, str(d.get("error")))
        if c["model"] == "op":
            check_op(c, ranks)
            continue
        for r, d in enumerate(ranks):  # the same bits on every rank: steps, parameters, the head's gradients, logits
            for k in ranks[0]:
                if k != "top":
                    assert np.array_equal(d[k], ranks[0][k]), (c["name"], r, k)
        res, want, logits = oracle(c)
        steps = ranks[0]["steps"]
        for t, w in enumerate(res):
            assert abs(steps[t][0] - w[0]) <= 1e-9 * abs(w[0]) and abs(steps[t][3] - w[3]) <= 1e-9 * abs(w[3]), (c["name"], t)
            assert (steps[t][1], steps[t][2]) == (w[1], w[2]), (c["name"], t)
        for k, w in want.items():
            assert _close(ranks[0][k], w, 1e-9), (c["name"], k)
        assert _close(ranks[0]["logits"], logits, 1e-9), c["name"]
