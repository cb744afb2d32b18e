"""Filtered link ranking on several ranks on the GPU (tests/mp_link_ranking_worker.py): R-GCN with a DistMult decoder
on the 1.5D dense shift with replication reuse at c = 1 and 2 and with local kernel fusion at c = 1, at p = 2 and 4.
The ranks and the MRR are bit-identical on every rank and across repeats, equal to p = 1's and equal to
tests/link_ranking_oracle.py's on the gathered output rows, copies of one row on different ranks tie exactly, and the
refusals (a layout without full rows, queries that differ on one rank, an id >= M on one rank) come on every rank.

Ranks share cuda:0 over the gloo-backed transport unless there is one GPU per rank (then NCCL)."""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from tests import link_ranking_oracle as lro
from tests.mp_link_ranking_worker import global_inputs, isolated
from tests.mp_util import ROOT, free_port

pytestmark = pytest.mark.gpu
SEED = 0xC0FFEE + 437
LOGM = 8


def case(alg, c, **kw):
    name = f"{alg}_c{c}_" + "_".join(f"{k}{v}" for k, v in sorted(kw.items()))
    return dict(name=name, alg=alg, c=c, logM=LOGM, seed=SEED, **kw)


LAYOUTS = [("15d_fusion1", 1), ("15d_fusion1", 2), ("15d_fusion2", 1)]
REFUSALS = {p: [case("15d_sparse", 1, expect="not defined"),
                case("15d_fusion1", 1, bad="queries", bad_rank=p - 1, expect="queries differ between ranks"),
                case("15d_fusion1", 1, bad="id", bad_rank=p - 1, expect="outside")] for p in (2, 4)}


def run(nproc, cases, timeout=900):
    transport = "nccl" if torch.cuda.device_count() >= nproc else "gloo"
    with tempfile.TemporaryDirectory() as td:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
               "--master-addr", "127.0.0.1", "--master-port", str(free_port()),
               os.path.join(ROOT, "tests", "mp_link_ranking_worker.py"), json.dumps(cases), td, transport]
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


@pytest.fixture(scope="module")
def single():
    c = case("15d_fusion1", 1)
    d = run(1, [c])[c["name"]][0]
    assert "error" not in d, str(d.get("error"))
    return d


def gathered_z(ranks, N):
    z = np.zeros((N, ranks[0]["z"].shape[1]))
    for d in ranks:
        top = int(d["top"][0])
        hi = min(top + len(d["z"]), N)
        if hi > top:
            z[top:hi] = d["z"][:hi - top]
    return z


@pytest.mark.parametrize("nproc", [2, 4])
def test_link_ranking_multirank(nproc, single):
    N = 1 << LOGM
    cases = [case(a, c) for a, c in LAYOUTS] + REFUSALS[nproc]
    got = run(nproc, cases)
    F, q, _, _, rel = global_inputs(cases[0])
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
            for k in ("tail", "head", "mrr"):
                assert np.array_equal(d[k], ranks[0][k]), (c["name"], r, k, "differs across ranks")
            assert np.array_equal(d["again"], np.concatenate([d["tail"], d["head"], d["mrr"]])), (c["name"], r)
        d0 = ranks[0]
        assert np.array_equal(d0["tail"], single["tail"]) and np.array_equal(d0["head"], single["head"]), c["name"]
        z = gathered_z(ranks, N)
        iso = isolated(N)
        assert np.array_equal(z[iso[0]], z[iso[1]]) and np.array_equal(z[iso[0]], z[iso[2]])
        owners = {int(i) * nproc // N for i in iso}
        assert len(owners) > 1  # the copies live on different ranks
        mrr, t, h, st, sh = lro.filtered_ranks(z, rel, q, [F], N)
        # the last two queries have the copies among their tail and head candidates: ties the equal ranks count
        assert st[-2][iso[0]] == st[-2][iso[1]] == st[-2][iso[2]] and sh[-1][iso[0]] == sh[-1][iso[1]] == sh[-1][iso[2]]
        assert np.array_equal(d0["tail"], t) and np.array_equal(d0["head"], h), c["name"]
        assert d0["mrr"][0] == pytest.approx(mrr, rel=1e-14)
