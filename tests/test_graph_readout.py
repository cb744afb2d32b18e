"""Graph-level prediction, CPU side: the fp64 oracle (tests/graph_readout_oracle.py) against a plain torch nn.Module
pipeline (index_add_ / scatter_reduce pooling, nn.Linear, F.cross_entropy, torch.optim.AdamW), its segment plan and
numpy kernels, and the new C and Python entry points refusing bad arguments without a GPU."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import graph_readout_oracle as gro
from tests import graph_sage_oracle as gso


class _Readout(torch.nn.Module):
    """The pipeline a torch user writes: pool by graph, then nn.Linear."""

    def __init__(self, r, C, pool, W, b):
        super().__init__()
        self.pool = pool
        self.lin = torch.nn.Linear(r, C, dtype=torch.float64)
        with torch.no_grad():
            self.lin.weight.copy_(torch.from_numpy(W.T))
            self.lin.bias.copy_(torch.from_numpy(b))

    def forward(self, H, batch, G):
        b = torch.as_tensor(batch)
        keep = b >= 0
        h, b = H[keep], b[keep]
        idx = b[:, None].expand(len(b), H.shape[1])
        if self.pool == "max":
            P = torch.zeros(G, H.shape[1], dtype=H.dtype).scatter_reduce(0, idx, h, "amax", include_self=False)
        else:
            P = torch.zeros(G, H.shape[1], dtype=H.dtype).index_add_(0, b, h)
            if self.pool == "mean":
                P = P / torch.bincount(b, minlength=G).clamp(min=1).to(H.dtype)[:, None]
        return self.lin(P)


def _batch(rng, N, G):
    batch = rng.integers(0, G, N)
    batch[rng.random(N) < 0.1] = -1
    batch[batch == 2] = 3  # graph 2 is empty
    return batch


@pytest.mark.parametrize("pool", gro.POOLS)
def test_oracle_matches_a_torch_module_pipeline(pool):
    rng = np.random.default_rng(1)
    N, G, r, Cc = 60, 7, 5, 3
    batch = _batch(rng, N, G)
    H = rng.standard_normal((N, r))
    W, b = rng.standard_normal((r, Cc)), rng.standard_normal(Cc)
    y = torch.from_numpy(rng.integers(0, Cc, G))
    y[4] = -1
    mod = _Readout(r, Cc, pool, W, b)
    Ht = torch.from_numpy(H).requires_grad_()
    loss = F.cross_entropy(mod(Ht, batch, G), y, ignore_index=-1)
    loss.backward()
    Ho = torch.from_numpy(H).requires_grad_()
    head = tuple(gro._t(v).requires_grad_() for v in (W, b))
    lo = F.cross_entropy(gro.head_torch(gro.pool_torch(Ho, batch, G, pool), head), y, ignore_index=-1)
    lo.backward()
    assert math.isclose(float(lo.detach()), float(loss.detach()), rel_tol=1e-14)
    # no ties in random data: the gradients agree too, max included
    assert torch.allclose(Ho.grad, Ht.grad, rtol=1e-13, atol=1e-15)
    assert torch.allclose(head[0].grad, mod.lin.weight.grad.T, rtol=1e-13, atol=1e-15)
    assert torch.allclose(head[1].grad, mod.lin.bias.grad, rtol=1e-13, atol=1e-15)


def test_max_splits_the_gradient_over_ties_and_signed_zeros():
    H = torch.tensor([[1.0, 0.0], [1.0, -0.0], [0.5, -1.0], [7.0, 7.0]], dtype=torch.float64, requires_grad=True)
    batch = np.array([0, 0, 0, 1])
    P = gro.pool_torch(H, batch, 3, "max")
    assert P.tolist() == [[1.0, 0.0], [7.0, 7.0], [0.0, 0.0]]
    P.backward(torch.ones_like(P))
    assert H.grad.tolist() == [[0.5, 0.5], [0.5, 0.5], [0.0, 0.0], [1.0, 1.0]]
    Pn, Cn = gro.pool_np(H.detach().numpy(), batch, 3, "max")
    assert Cn.tolist() == [[2, 2], [1, 1], [0, 0]] and np.isneginf(Pn[2]).all()
    dH = gro.pool_grad_np(batch, 3, np.ones((3, 2)), H=H.detach().numpy(), P=np.where(Cn == 0, 0, Pn), C=Cn)
    assert np.array_equal(dH, H.grad.numpy())


def test_plan_chunks_segments_and_keeps_rows_ascending():
    rng = np.random.default_rng(2)
    G = 5
    batch = np.concatenate([np.full(600, 1), np.full(3, 4), np.full(256, 3), [-1, -1]])
    rng.shuffle(batch)
    seg_start, seg_rows, chunk_first, chunk_seg = gro.plan(batch, G)
    assert np.diff(seg_start).tolist() == [0, 600, 0, 256, 3]
    assert np.diff(chunk_first).tolist() == [1, 3, 1, 1, 1] and chunk_first[-1] == len(chunk_seg)
    assert chunk_seg.tolist() == [0, 1, 1, 1, 2, 3, 4]
    for g in range(G):
        rows = seg_rows[seg_start[g]:seg_start[g + 1]]
        assert (np.diff(rows) > 0).all() and (batch[rows] == g).all()


def test_training_oracle_equals_a_torch_loop():
    """gro.train on GraphSAGE's model equals a hand-written loop with nn.Linear and torch.optim.AdamW."""
    rng = np.random.default_rng(3)
    N, G, layers, Cc = 30, 4, [(3, 4)], 2
    rows, cols = rng.integers(0, N, 90), rng.integers(0, N, 90)
    params = gso.random_params(layers, rng)
    X = gso._t(rng.standard_normal((N, 3)))
    batch = rng.integers(0, G, N)
    labels = np.array([0, 1, -1, 1])
    W, b = rng.standard_normal((4, Cc)), rng.standard_normal(Cc)
    tp = gso._leaves(params)
    res, head = gro.train(lambda _: gso.model_torch(rows, cols, N, layers, tp, X, "sum"), [v for P in tp for v in P.values()],
                          batch, G, "max", (W, b), labels, 3, lr=0.05)
    tq = gso._leaves(params)
    mod = _Readout(4, Cc, "max", W, b)
    opt = torch.optim.AdamW([v for P in tq for v in P.values()] + [mod.lin.weight, mod.lin.bias], lr=0.05, foreach=False)
    for t in range(3):
        opt.zero_grad()
        loss = F.cross_entropy(mod(gso.model_torch(rows, cols, N, layers, tq, X, "sum"), batch, G), torch.from_numpy(labels),
                               ignore_index=-1)
        loss.backward()
        assert math.isclose(float(loss.detach()), res[t][0], rel_tol=1e-12) and res[t][2] == 3
        opt.step()
    assert np.allclose(head[0], mod.lin.weight.detach().numpy().T, rtol=1e-11, atol=1e-14)
    for P, Q in zip(tp, tq):
        for k in P:
            assert np.allclose(P[k].detach().numpy(), Q[k].detach().numpy(), rtol=1e-11, atol=1e-14), k


def test_readout_kernels_validate_without_a_gpu(hnh):
    bufs = [(C.c_double * 64)() for _ in range(8)]
    ss, sr, cf, cs, h, p, c, ws = (C.addressof(b) for b in bufs)

    def pool(ss=ss, sr=sr, cf=cf, cs=cs, segs=2, chunks=2, h=h, ldh=4, r=4, p=p, ldp=4, c=None, ldc=4, ws=None, wsb=0):
        return hnh.hnh_segment_pool_f64(ss, sr, cf, cs, segs, chunks, h, ldh, r, p, ldp, c, ldc, ws, wsb, None)

    err = lambda: hnh.hnh_last_error_string()  # noqa: E731
    assert pool(segs=-1) == -1 and b"count" in err()
    assert pool(chunks=1) == -1 and b"count" in err()
    assert pool(r=0) == -1 and b"r must be positive" in err()
    for kw in (dict(ldh=3), dict(ldp=3), dict(c=c, ldc=3)):
        assert pool(**kw) == -1 and b"leading dimension" in err(), kw
    for k in ("ss", "cf", "cs", "h", "p"):
        assert pool(**{k: None}) == -1 and b"null" in err(), k
    assert pool(p=h) == -1 and b"may not be the input" in err()
    assert pool(c=p) == -1 and b"distinct" in err()
    assert pool(chunks=3) == -1 and b"workspace" in err()
    assert pool(segs=0, chunks=0, ss=None) == 0  # nothing to pool
    assert hnh.hnh_segment_pool_workspace_bytes(3, 4, 1) == 3 * 4 * 2 * 8 and hnh.hnh_segment_pool_workspace_bytes(-1, 4, 0) == -1

    def grad(rg=ss, rows=4, graphs=2, dp=p, lddp=4, scale=None, h=None, ldh=4, pp=None, ldp=4, c=None, ldc=4, r=4, dh=ws, lddh=4):
        return hnh.hnh_segment_pool_grad_f64(rg, rows, graphs, dp, lddp, scale, h, ldh, pp, ldp, c, ldc, r, dh, lddh, None)

    assert grad(rows=-1) == -1 and b"negative" in err()
    assert grad(r=0) == -1
    assert grad(h=h) == -1 and b"together" in err()
    assert grad(h=h, pp=p, c=c, scale=cs) == -1 and b"no scale" in err()
    assert grad(lddh=3) == -1 and b"leading dimension" in err()
    assert grad(rg=None) == -1 and b"null" in err()
    assert grad(dh=p) == -1 and b"may not be an input" in err()
    assert grad(rows=0) == 0
    assert hnh.hnh_segment_max_count_merge_f64(c, p, h, -1, None) == -1
    assert hnh.hnh_segment_max_count_merge_f64(None, p, h, 4, None) == -1
    assert hnh.hnh_segment_max_count_merge_f64(p, p, h, 4, None) == -1
    assert hnh.hnh_segment_max_count_merge_f64(None, None, None, 0, None) == 0
    if not torch.cuda.is_available():  # no CPU fallback: compute fails with HNH_E_CUDA
        assert pool() == -2 and grad() == -2


def test_readout_entry_points_validate_without_a_gpu(hnh):
    out = C.c_void_p()
    res = (C.c_double * 4)()
    p = C.addressof(res)
    batch = (C.c_int64 * 4)()
    assert hnh.hnhd_readout_create(None, batch, 4, 2, b"sum", 0, C.byref(out)) == -1 and b"null" in hnh.hnh_last_error_string()
    assert hnh.hnhd_readout_create(p, batch, 4, 2, None, 0, C.byref(out)) == -1
    assert hnh.hnhd_readout_create(p, batch, 4, 2, b"sum", 0, None) == -1
    for args in ((None, p, p), (p, None, p), (p, p, None)):
        assert hnh.hnhd_readout_pool(*args) == -1 and b"null" in hnh.hnh_last_error_string()
    assert hnh.hnhd_readout_pool_backward(p, p, p, None) == -1 and hnh.hnhd_readout_pool_backward(None, p, p, p) == -1
    assert hnh.hnhd_readout_pool_backward(p, p, C.c_void_p(p + 8), p) == -1 and b"dH may not" in hnh.hnh_last_error_string()
    r, c = C.c_int64(), C.c_int64()
    assert hnh.hnhd_readout_param_shape(None, b"weight", C.byref(r), C.byref(c)) == -1
    assert hnh.hnhd_readout_param_shape(p, None, C.byref(r), C.byref(c)) == -1
    for f in (hnh.hnhd_readout_set_param, hnh.hnhd_readout_get_param, hnh.hnhd_readout_get_param_grad):
        assert f(None, b"bias", p) == -1
    assert hnh.hnhd_graph_labels_create(None, batch, 4, 2, C.byref(out)) == -1 and hnh.hnhd_graph_labels_create(p, batch, 4, 2, None) == -1
    for args in ((None, p, p, p), (p, None, p, p), (p, p, None, p), (p, p, p, None)):
        assert hnh.hnhd_model_graph_train_step(*args, 0.0, 0, res) == -1 and b"null" in hnh.hnh_last_error_string()
    assert hnh.hnhd_model_graph_train_step(p, p, p, p, 0.0, 0, None) == -1
    for args in ((None, p, p), (p, None, p), (p, p, None)):
        assert hnh.hnhd_model_graph_evaluate(*args, None, res) == -1
    assert hnh.hnhd_model_graph_evaluate(p, p, p, None, None) == -1
    hnh.hnhd_readout_destroy(None)
    hnh.hnhd_graph_labels_destroy(None)


def test_python_front_end_validates_graph_arguments():
    from distributed_sddmm_b200 import driver as D
    net = D.GraphSAGE.__new__(D.GraphSAGE)
    net.h, net.layers = None, [(3, 4)]
    with pytest.raises(ValueError, match="1-D integer array"):
        D.GraphReadout(net, np.zeros(4), 2)
    with pytest.raises(ValueError, match="pool"):
        D.GraphReadout(net, np.zeros(4, np.int64), 2, pool="attention")
    with pytest.raises(ValueError, match="num_graphs"):
        D.GraphReadout(net, np.zeros(4, np.int64), 2.5)
    with pytest.raises(ValueError, match="num_classes"):
        D.GraphReadout(net, np.zeros(4, np.int64), 2, num_classes=0)
    with pytest.raises(RuntimeError, match="readout_create failed"):
        D.GraphReadout(net, np.zeros(4, np.int64), 2, num_classes=3)  # null model handle
    with pytest.raises(TypeError, match="GraphReadout"):
        D.GraphLabels(None, [0, 1], 2)
    ro = D.GraphReadout.__new__(D.GraphReadout)
    ro.h, ro._H = None, None
    with pytest.raises(ValueError, match="1-D integer array"):
        D.GraphLabels(ro, [0.5, 1.0], 2)
    with pytest.raises(ValueError, match="num_classes"):
        D.GraphLabels(ro, [0, 1], None)
    with pytest.raises(RuntimeError, match="graph_labels_create failed"):
        D.GraphLabels(ro, [0, 1], 2)
    with pytest.raises(TypeError, match="H must be a Dense"):
        ro.pool(np.zeros((4, 4)))
    dense = D.Dense.__new__(D.Dense)
    dense.h = None
    with pytest.raises(ValueError, match="pool first"):
        ro.pool_backward(dense)
    opt = D.AdamW()
    labels = D.GraphLabels.__new__(D.GraphLabels)
    labels.h = None
    for m in (net, D.GAT.__new__(D.GAT), D.GraphTransformer.__new__(D.GraphTransformer), D.RGCN.__new__(D.RGCN)):
        m.h = None
        with pytest.raises(TypeError, match="GraphReadout"):
            m.graph_train_step(None, labels, opt)
        with pytest.raises(TypeError, match="GraphLabels"):
            m.graph_train_step(ro, None, opt)
        with pytest.raises(TypeError, match="AdamW"):
            m.graph_train_step(ro, labels, None)
        with pytest.raises(TypeError, match="GraphReadout"):
            m.graph_evaluate(object(), labels)
    gt = D.GraphTransformer.__new__(D.GraphTransformer)
    gt.h = None
    with pytest.raises(ValueError, match="dropout"):
        gt.graph_train_step(ro, labels, opt, dropout=1.0)
