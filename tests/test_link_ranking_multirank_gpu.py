"""Filtered link ranking on several ranks on the GPU (tests/mp_link_ranking_worker.py): R-GCN with a DistMult decoder
on the 1.5D dense shift with replication reuse at c = 1 and 2 and with local kernel fusion at c = 1, at p = 2 and 4.
The ranks and the MRR are bit-identical on every rank and across repeats, equal to p = 1's and equal to
tests/link_ranking_oracle.py's on the gathered output rows, copies of one row on different ranks tie exactly, and the
refusals (a layout without full rows, queries that differ on one rank, an id >= M on one rank) come on every rank.
Then a GraphSAGE r = 65536 wide with integer outputs, ranked in three query chunks, at M = 301 (the last rank holds
padding rows) and, at p = 4, M = 9 (the last rank holds no valid row), with large values in every padding row: the
ranks equal p = 1's and the exact oracle's on the gathered output; and a GAT and a GINE on the float path.

Ranks share cuda:0 over the gloo-backed transport unless there is one GPU per rank (then NCCL)."""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

from tests import link_ranking_cases as lrc
from tests import link_ranking_oracle as lro
from tests import mp_link_ranking_worker as mlw
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


# ---- other models, any M: padding rows, an empty rank, several query chunks ---------------------------------------------
WIDE_R, WIDE_NQ = 65536, 2 * 256 + 5  # three query chunks: 256, 256 and 5


def model_case(alg, c, model, M, **kw):
    extra = dict(r=WIDE_R, n_q=WIDE_NQ, pad=1000.0) if model == "sage_wide" else dict(pad=1000.0)
    extra.update(kw)
    return dict(name=f"{model}_M{M}_{alg}_c{c}", alg=alg, c=c, model=model, M=M, seed=SEED + 5, **extra)


WIDE_M = {2: [301], 4: [301, 9]}
MODEL_CASES = {p: [model_case(a, c, "sage_wide", M) for M in WIDE_M[p] for a, c in LAYOUTS] +
               [model_case("15d_fusion1", 1, m, 301) for m in ("gat", "gine")] for p in (2, 4)}


@pytest.fixture(scope="module")
def single_models():
    """p = 1 runs of every model case, by (model, M)."""
    cases = {(c["model"], c["M"]): model_case("15d_fusion1", 1, c["model"], c["M"]) for p in MODEL_CASES for c in MODEL_CASES[p]}
    got = run(1, list(cases.values()))
    out = {}
    for key, c in cases.items():
        d = got[c["name"]][0]
        assert "error" not in d, (c["name"], str(d.get("error")))
        out[key] = d
    return out


def padding_outranks(ranks, case, F, q, rel):
    """The share of queries (nonzero query vector) some padding row in the output buffers would outscore the true
    entity for, in the tail and the head direction, and the number of padding rows."""
    M = case["M"]
    pads = np.concatenate([d["z"][max(0, M - int(d["top"][0])):] for d in ranks])
    z = gathered_z(ranks, M)
    shares = []
    for a, b in ((q[0], q[2]), (q[2], q[0])):
        Q = z[a] * rel[q[1]]
        true = (Q * z[b]).sum(1)
        live = np.abs(Q).sum(1) > 0
        shares.append(((Q @ pads.T).max(1) > true)[live].mean())
    return shares, len(pads)


@pytest.mark.parametrize("nproc", [2, 4])
def test_link_ranking_multirank_models_padding_and_chunks(nproc, single_models):
    got = run(nproc, MODEL_CASES[nproc])
    for c in MODEL_CASES[nproc]:
        ranks, M = got[c["name"]], c["M"]
        for r, d in enumerate(ranks):
            assert "error" not in d, (c["name"], r, str(d.get("error")))
            for k in ("tail", "head", "mrr"):
                assert np.array_equal(d[k], ranks[0][k]), (c["name"], r, k, "differs across ranks")
            assert np.array_equal(d["again"], np.concatenate([d["tail"], d["head"], d["mrr"]])), (c["name"], r)
        d0, one = ranks[0], single_models[(c["model"], M)]
        assert np.array_equal(d0["tail"], one["tail"]) and np.array_equal(d0["head"], one["head"]), c["name"]
        tops = [int(d["top"][0]) for d in ranks]
        blocks = lrc.block_rows(M, nproc)
        assert sorted(tops) == [b[0] for b in blocks], (c["name"], tops)  # the blocks, in the grid's rank order
        (_, F, q, _, _, rel) = mlw.model_inputs(c)
        z = gathered_z(ranks, M)
        if c["model"] != "sage_wide":
            mrr, t, h, st, sh = lro.matmul_ranks(z, np.ones((1, z.shape[1])), q, [F], M)
            assert lro.separated(st, sh, q), c["name"]
            assert np.array_equal(d0["tail"], t) and np.array_equal(d0["head"], h), c["name"]
            continue
        assert np.array_equal(z, gathered_z([one], M))  # integer-valued: the same output at any p
        iso = lrc.isolated(M)
        assert all(np.array_equal(z[iso[0]], z[i]) for i in iso[1:])
        assert np.array_equal(z, np.round(z)) and lro.integer_bound(z, rel) < 2.0 ** 43
        mrr, t, h, _, _ = lro.matmul_ranks(z, rel, q, [F], M)
        assert np.array_equal(d0["tail"], t) and np.array_equal(d0["head"], h), c["name"]
        assert d0["mrr"][0] == pytest.approx(mrr, rel=1e-14)
        # the padding rows hold X_pad W + b, far above every real row: counted, they would outrank the true entity
        shares, n_pad = padding_outranks(ranks, c, F, q, rel)
        assert n_pad == nproc * blocks[0][1] - M > 0 and min(shares) == 1.0, (c["name"], shares, n_pad)
