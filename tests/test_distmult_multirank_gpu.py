"""Relational link prediction on several ranks on the GPU (tests/mp_distmult_worker.py), on the 1.5D dense shift with
replication reuse at c = 1 and 2 and with local kernel fusion at c = 1, at p = 2 and 4: the op (a positive call and an
accumulated negative one, H_A = H_B, dH_A = dH_B, dD and scores) against tests/distmult_oracle.py with the sums and dD
bit-identical on every rank and repeats bit-identical; 3 relational link train steps of R-GCN, plain and with bases,
with every parameter and the relation table bit-identical on every rank and within 1e-9 of the oracle's global run; and
refusals on every rank (a layout without full rows, a relation out of range on one rank only).

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
from tests import distmult_oracle as dmo
from tests import rgcn_basis_oracle as bo
from tests import rgcn_oracle as ro
from tests.mp_distmult_worker import LAYERS, R, global_inputs, s_relations
from tests.mp_util import ROOT, free_port

pytestmark = pytest.mark.gpu


def case(model, alg, c, steps=3, logM=7, seed=0xC0FFEE + 419, **kw):
    base = dict(r=8)
    base.update(kw)
    name = f"{model}_{alg}_c{c}_" + "_".join(f"{k}{v}" for k, v in sorted(kw.items()))
    return dict(name=name, model=model, alg=alg, c=c, steps=steps, logM=logM, seed=seed, **base)


LAYOUTS = [("15d_fusion1", 1), ("15d_fusion1", 2), ("15d_fusion2", 1)]
CASES = {
    p: [case("op", a, c) for a, c in LAYOUTS] + [case("op", "15d_fusion1", 1, r=7)]
    + [case("train", a, c) for a, c in LAYOUTS] + [case("train", "15d_fusion1", 2, bases=2)]
    + [case("op", "15d_sparse", 1, expect="not defined"), case("op", "15d_fusion2", 2, expect="not defined"),
       case("train", "15d_fusion1", 1, bad_rank=p - 1, expect="not integers in")]
    for p in (2, 4)
}


def run(nproc, cases, timeout=900):
    transport = "nccl" if torch.cuda.device_count() >= nproc else "gloo"
    with tempfile.TemporaryDirectory() as td:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
               "--master-addr", "127.0.0.1", "--master-port", str(free_port()),
               os.path.join(ROOT, "tests", "mp_distmult_worker.py"), json.dumps(cases), td, transport]
        env = dict(os.environ, OMP_NUM_THREADS="2")
        p = subprocess.run(cmd, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=timeout, text=True)
        if p.returncode != 0 and "Address already in use" in p.stdout:
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


def _scores_match(got, er, ec, trip, want):
    g, w = {}, {}
    for s, u, v in zip(got, er, ec):
        g.setdefault((u, v), []).append(s)
    for s, u, v in zip(want, trip[0], trip[1]):
        w.setdefault((u, v), []).append(s)
    return all(k in w and _close(np.sort(g[k]), np.sort(w[k]), 1e-12) for k in g)


def check_op(c, ranks):
    N = 1 << c["logM"]
    pos, neg, H, rel, _, _ = global_inputs(c)
    inv = 1.0 / (len(pos[0]) + len(neg[0]))
    lp, cp, sp, gp, _, dp = dmo.op(H, H, rel, *pos, 1.0, inv, same=True)
    ln, cn, sn, gn, _, dn = dmo.op(H, H, rel, *neg, 0.0, inv, same=True)
    for r, d in enumerate(ranks):
        assert np.array_equal(d["res"], ranks[0]["res"]) and np.array_equal(d["res"][:2], d["res"][2:]), (c["name"], r)
        assert np.array_equal(d["dD"], ranks[0]["dD"]), (c["name"], r, "dD differs across ranks")
        top = int(d["top"][0])
        hi = min(top + len(d["dH"]), N)
        assert _close(d["dH"][:hi - top], (gp + gn)[top:hi], 1e-12), (c["name"], r)
        assert _scores_match(d["sp"], d["erp"], d["ecp"], pos, sp) and _scores_match(d["sn"], d["ern"], d["ecn"], neg, sn)
    res = ranks[0]["res"]
    assert abs(res[0][0] - lp) <= 1e-12 * lp and abs(res[1][0] - ln) <= 1e-12 * ln
    assert abs(res[0][1] - cp) <= 2 and abs(res[1][1] - cn) <= 2
    assert _close(ranks[0]["dD"], dp + dn, 1e-12)


def oracle(c):
    N = 1 << c["logM"]
    rows, cols, _ = orc.er_tuples(c["logM"], 5, c["seed"])
    rows, cols = np.asarray(rows, np.int64), np.asarray(cols, np.int64)
    rels = s_relations(rows, cols, N)
    pos, neg, _, rel, params, X = global_inputs(c)
    rel0 = rel[:, :LAYERS[-1][1]]
    if c.get("bases"):
        params = bo.random_params(LAYERS, R, c["bases"], np.random.default_rng(c["seed"] + 9))
        fwd = lambda tp, x: bo.model_torch(rows, cols, rels, N, LAYERS, tp, x, R, c["bases"], "mean")  # noqa: E731
    else:
        fwd = lambda tp, x: ro.model_torch(rows, cols, rels, N, LAYERS, tp, x, R, "mean")  # noqa: E731
    tp = [{k: dmo._t(v).clone().requires_grad_() for k, v in P.items()} for P in params]
    x = dmo._t(X)
    res, rel_t = dmo.train(lambda _: fwd(tp, x), [v for P in tp for v in P.values()], rel0, pos, neg, c["steps"], lr=1e-2,
                           max_grad_norm=1.0)
    want = {f"p{l}_{k}": v.detach().numpy() for l, P in enumerate(tp) for k, v in P.items()}
    want["rel"] = rel_t
    return res, want


@pytest.mark.parametrize("nproc", [2, 4])
def test_distmult_multirank(nproc):
    cases = CASES[nproc]
    got = run(nproc, cases)
    for c in cases:
        ranks = got[c["name"]]
        if c.get("expect"):
            for r, d in enumerate(ranks):
                assert "error" in d, (c["name"], r)
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
            assert int(steps[t][2]) == w[2] and abs(int(steps[t][1]) - w[1]) <= 1, (c["name"], t)
        for k, w in want.items():
            assert _close(ranks[0][k], w, 1e-9), (c["name"], k, np.abs(ranks[0][k] - w).max())
