"""Link prediction on several ranks on the GPU (tests/mp_link_prediction_worker.py), on the 1.5D dense shift with
replication reuse at c = 1 and 2 and with local kernel fusion at c = 1, at p = 2 and 4: the op (H_A = H_B, dH_A = dH_B,
scores) against tests/link_prediction_oracle.py with loss and correct count equal on every rank and repeats
bit-identical; 3 link train steps of the graph transformer (blocks, gate, edge features, dropout, clipping) and of GAT,
with the parameters bit-identical on every rank and within 1e-9 of the oracle's global run; and refusals on every rank
(layouts without full rows, a T of another c or algorithm, a bad target on one rank only).

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
from tests import link_prediction_oracle as lpo
from tests.mp_graph_transformer_worker import attr_of
from tests.mp_link_prediction_worker import GAT_LAYERS, GT_LAYERS, global_inputs
from tests.mp_util import ROOT, free_port

pytestmark = pytest.mark.gpu


def case(model, alg, c, steps=3, logM=7, seed=0xC0FFEE + 181, **kw):
    base = dict(r=16, dropout=0.3 if model == "gt" else 0.0, clip=0.05 if model == "gt" else None, kind="additive")
    base.update(kw)
    name = f"{model}_{alg}_c{c}_" + "_".join(f"{k}{v}" for k, v in sorted(kw.items()))
    return dict(name=name, model=model, alg=alg, c=c, steps=steps, logM=logM, seed=seed, **base)


LAYOUTS = [("15d_fusion1", 1), ("15d_fusion1", 2), ("15d_fusion2", 1)]
CASES = {
    p: [case("op", a, c) for a, c in LAYOUTS] + [case("op", "15d_fusion1", 1, r=7)]
    + [case("gt", a, c) for a, c in LAYOUTS] + [case("gat", "15d_fusion1", 2), case("gat", "15d_fusion2", 1, kind="softmax")]
    + [case("op", "15d_sparse", 1, expect="not defined"), case("op", "15d_fusion2", 2, expect="not defined"),
       case("gt", "15d_fusion1", 1, t_c=2, expect="layout"), case("gt", "15d_fusion1", 1, t_alg="15d_fusion2", expect="layout"),
       case("gt", "15d_fusion1", 1, bad_rank=p - 1, expect="[0, 1]")]
    + ([case("op", "25d_dense_replicate", 1, expect="not defined")] if p == 4 else [])
    for p in (2, 4)
}


def run(nproc, cases, timeout=900):
    """Returns {case name: [per-rank dict]}."""
    transport = "nccl" if torch.cuda.device_count() >= nproc else "gloo"
    with tempfile.TemporaryDirectory() as td:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
               "--master-addr", "127.0.0.1", "--master-port", str(free_port()),
               os.path.join(ROOT, "tests", "mp_link_prediction_worker.py"), json.dumps(cases), td, transport]
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


def check_op(c, ranks):
    N = 1 << c["logM"]
    tr, tc, y, H, _, _ = global_inputs(c)
    wl, wc, wn, ws, wg, _ = lpo.link_loss(H, H, tr, tc, y, same=True)
    score_of = {(u, v): s for u, v, s in zip(tr, tc, ws)}
    for r, d in enumerate(ranks):
        assert np.array_equal(d["res"], ranks[0]["res"]) and np.array_equal(d["again"], d["res"]), (c["name"], r)
        top = int(d["top"][0])
        hi = min(top + len(d["dH"]), N)
        assert np.abs(d["dH"][:hi - top] - wg[top:hi]).max() <= 1e-12 * np.abs(wg).max(), (c["name"], r)
        assert not d["dH"][hi - top:].any()
        want = np.array([score_of[(u, v)] for u, v in zip(d["er"], d["ec"])])
        assert np.abs(d["scores"] - want).max() <= 1e-12 * max(np.abs(want).max(), 1.0), (c["name"], r)
    loss, correct, count = ranks[0]["res"]
    assert abs(loss - wl) <= 1e-12 * wl and count == wn and abs(correct - wc) <= 2, (c["name"], ranks[0]["res"], wl, wc)


def oracle(c):
    N = 1 << c["logM"]
    rows, cols, _ = orc.er_tuples(c["logM"], 5, c["seed"])
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    tr, tc, y, _, params, X = global_inputs(c)
    if c["model"] == "gt":
        res, trained = lpo.train_gt(rows, cols, N, GT_LAYERS, params, X, (tr, tc, y), c["steps"], attr=attr_of(rows, cols, 2),
                                    beta=True, ffn=1, dropout=c["dropout"], seeds=[5 + t for t in range(c["steps"])], lr=1e-2,
                                    max_grad_norm=c["clip"])
        return res, {f"p{l}_{k}": v for l, P in enumerate(trained) for k, v in P.items()}
    res, ws, u1, u2 = lpo.train_gat(c["kind"], rows, cols, N, GAT_LAYERS, *params, X, (tr, tc, y), c["steps"], lr=1e-2)
    want = {}
    for l, (_, _, H) in enumerate(GAT_LAYERS):
        for h in range(H):
            want[f"w{l}_{h}"], want[f"a1_{l}_{h}"], want[f"a2_{l}_{h}"] = ws[l][h], u1[l][h], u2[l][h]
    return res, want


@pytest.mark.parametrize("nproc", [2, 4])
def test_link_prediction_multirank(nproc):
    cases = CASES[nproc]
    got = run(nproc, cases)
    for c in cases:
        ranks = got[c["name"]]
        if c.get("expect"):
            for r, d in enumerate(ranks):
                assert "error" in d and "code -1" in str(d["error"]), (c["name"], r, {k: v for k, v in d.items() if k == "error"})
                msg = str(d["error"])
                assert c["expect"] in msg or (c.get("bad_rank") is not None and "another rank" in msg), (c["name"], r, msg)
            continue
        for r, d in enumerate(ranks):
            assert "error" not in d, (c["name"], r, str(d.get("error")))
        if c["model"] == "op":
            check_op(c, ranks)
            continue
        for r, d in enumerate(ranks):
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
