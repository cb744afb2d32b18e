"""Training, CPU side: the fp64 training oracle reproduces torch's own nn.Module training of the same model, and the new
C entry points, driver entry points and Python front end refuse bad arguments without a GPU (and fail cleanly when
asked to compute without one)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import graph_transformer_block_oracle as gbo
from tests import graph_transformer_oracle as gto
from tests import training_oracle as tro
from tests.test_sparse_attention_bias import _pattern


class _Layer(torch.nn.Module):
    """A TransformerConv layer with a post-norm block, written with torch's own modules (Linear weights out x in)."""

    def __init__(self, f, d, H, ffn):
        super().__init__()
        r = d * H
        self.f, self.d, self.H = f, d, H
        for n in gto.PROJECTIONS:
            setattr(self, "lin_" + n, torch.nn.Linear(f, r).double())
        self.norm1, self.norm2 = torch.nn.LayerNorm(r).double(), torch.nn.LayerNorm(r).double()
        self.lin1, self.lin2 = torch.nn.Linear(r, ffn * r).double(), torch.nn.Linear(ffn * r, r).double()

    def library_params(self):
        p = {}
        for n in gto.PROJECTIONS:
            lin = getattr(self, "lin_" + n)
            p[n], p[n + "_bias"] = lin.weight.detach().numpy().T.copy(), lin.bias.detach().numpy().copy()
        p["norm1"], p["norm1_bias"] = self.norm1.weight.detach().numpy().copy(), self.norm1.bias.detach().numpy().copy()
        p["norm2"], p["norm2_bias"] = self.norm2.weight.detach().numpy().copy(), self.norm2.bias.detach().numpy().copy()
        p["ffn1"] = np.vstack([self.lin1.weight.detach().numpy().T, self.lin1.bias.detach().numpy()])
        p["ffn2"] = np.vstack([self.lin2.weight.detach().numpy().T, self.lin2.bias.detach().numpy()])
        return p

    def forward(self, rows, cols, N, x):
        tp = {n: getattr(self, "lin_" + n).weight.T for n in gto.PROJECTIONS}
        tp.update({n + "_bias": getattr(self, "lin_" + n).bias for n in gto.PROJECTIONS})
        y = gto.model_torch(rows, cols, N, [(self.f, self.d, self.H)], [tp], x)
        h = self.norm1(y)
        return self.norm2(h + self.lin2(torch.relu(self.lin1(h))))


def test_oracle_reproduces_torch_module_training():
    """tests/training_oracle.py on the library's parameter layout follows torch's nn.Module training (AdamW over
    model.parameters(), clip_grad_norm_, cross_entropy with ignore_index) step for step."""
    rng = np.random.default_rng(5)
    N, layers, steps = 17, [(5, 3, 2), (6, 4, 1)], 4
    rows, cols = _pattern(rng, N, N, per_row=3)
    torch.manual_seed(0)
    mods = torch.nn.ModuleList([_Layer(f, d, H, 2) for f, d, H in layers])
    with torch.no_grad():
        for m in mods:
            for k in ("norm1", "norm2"):
                getattr(m, k).weight.uniform_(0.5, 1.5)
                getattr(m, k).bias.uniform_(-0.5, 0.5)
    params = [m.library_params() for m in mods]
    X = rng.standard_normal((N, 5))
    labels = rng.integers(-1, 4, N)
    kw = dict(lr=3e-2, weight_decay=0.05, max_grad_norm=0.5)
    want, trained = tro.train_gt(rows, cols, N, layers, params, X, labels, steps, ffn=2, **kw)

    opt = torch.optim.AdamW(mods.parameters(), lr=3e-2, weight_decay=0.05)
    lab = torch.from_numpy(labels.astype(np.int64))
    for t in range(steps):
        opt.zero_grad()
        out = gto._t(X)
        for m in mods:
            out = m(rows, cols, N, out)
        loss = F.cross_entropy(out, lab, ignore_index=-1)
        loss.backward()
        norm = torch.nn.utils.clip_grad_norm_(mods.parameters(), 0.5)
        assert math.isclose(float(loss), want[t][0], rel_tol=1e-12) and math.isclose(float(norm), want[t][3], rel_tol=1e-12)
        opt.step()
    for m, P in zip(mods, trained):
        for k, v in m.library_params().items():
            assert np.allclose(v, P[k], rtol=1e-11, atol=1e-12), k


def test_oracle_no_labelled_row_is_zero():
    """With no labelled row the oracle's loss and gradient are 0 (torch's mean would be NaN), so AdamW applies only the
    decay."""
    rng = np.random.default_rng(2)
    N, layers = 9, [(3, 2, 2)]
    rows, cols = _pattern(rng, N, N, per_row=2)
    params = gbo.random_params(layers, 0, False, 0, rng)
    res, trained = tro.train_gt(rows, cols, N, layers, params, rng.standard_normal((N, 3)), -np.ones(N), 2, lr=0.1)
    assert [r[0] for r in res] == [0.0, 0.0] and [r[3] for r in res] == [0.0, 0.0]
    assert np.allclose(trained[0]["query"], params[0]["query"] * (1 - 0.1 * 1e-2) ** 2, rtol=1e-15)


def test_training_kernels_validate_without_a_gpu(hnh):
    bufs = [(C.c_double * 64)() for _ in range(6)]
    a, b, c, d, e, w = (C.addressof(x) for x in bufs)
    lab = C.addressof((C.c_int32 * 8)())
    assert hnh.hnh_cross_entropy_workspace_bytes(-1) == -1
    ws = hnh.hnh_cross_entropy_workspace_bytes(1000)
    assert ws >= 8 * 2 * 1000 and hnh.hnh_cross_entropy_workspace_bytes(0) >= 0

    def ce(dl=a, sums=b, lg=c, lb=lab, n=4, Cc=4, ld=4, inv=0.25, ws_p=w, ws_bytes=1 << 20):
        return hnh.hnh_cross_entropy_f64(dl, sums, lg, lb, n, Cc, ld, inv, ws_p, ws_bytes, None)

    assert ce(n=-1) == -1 and b"negative" in hnh.hnh_last_error_string()
    assert ce(Cc=0) == -1 and b"class count" in hnh.hnh_last_error_string()
    assert ce(ld=3) == -1 and b"ld" in hnh.hnh_last_error_string()
    for bad in (-1.0, math.nan, math.inf):
        assert ce(inv=bad) == -1 and b"inv_count" in hnh.hnh_last_error_string()
    for k in ("dl", "sums", "lg", "lb"):
        assert ce(**{k: None}) == -1 and b"null" in hnh.hnh_last_error_string(), k
    assert ce(dl=c) == -1 and b"may not be" in hnh.hnh_last_error_string()
    assert ce(sums=a) == -1 and b"may not be" in hnh.hnh_last_error_string()
    assert ce(ws_p=None) == -1 and b"workspace" in hnh.hnh_last_error_string()
    assert ce(ws_bytes=hnh.hnh_cross_entropy_workspace_bytes(4) - 1) == -1

    def adamw(p=a, m=b, v=c, g=d, n=4, lr=1e-3, b1=0.9, b2=0.999, eps=1e-8, wd=0.0, bc1=0.1, bc2=0.001, clip=None):
        return hnh.hnh_adamw_f64(p, m, v, g, n, lr, b1, b2, eps, wd, bc1, bc2, clip, None)

    assert adamw(n=-1) == -1 and b"negative" in hnh.hnh_last_error_string()
    for kw in (dict(lr=-1.0), dict(lr=math.nan), dict(lr=math.inf), dict(b1=1.0), dict(b2=-0.1), dict(b1=math.nan),
               dict(eps=0.0), dict(eps=math.inf), dict(wd=-0.1), dict(wd=math.nan), dict(bc1=0.0), dict(bc2=1.5)):
        assert adamw(**kw) == -1, kw
    for k in ("p", "m", "v", "g"):
        assert adamw(**{k: None}) == -1 and b"null" in hnh.hnh_last_error_string(), k
    assert adamw(m=a) == -1 and b"distinct" in hnh.hnh_last_error_string()
    assert adamw(clip=d) == -1 and b"distinct" in hnh.hnh_last_error_string()
    assert adamw(n=0, p=None, m=None, v=None, g=None) == 0

    assert hnh.hnh_clip_coef_f64(a, b, -1, 1.0, None) == -1
    for bad in (-1.0, math.nan):
        assert hnh.hnh_clip_coef_f64(a, b, 2, bad, None) == -1 and b"max_norm" in hnh.hnh_last_error_string()
    assert hnh.hnh_clip_coef_f64(None, b, 2, 1.0, None) == -1 and hnh.hnh_clip_coef_f64(a, None, 2, 1.0, None) == -1
    if not torch.cuda.is_available():  # no CPU fallback: compute fails with HNH_E_CUDA
        assert ce() == -2
        assert ce(n=0) == -2  # the zero fill of sums needs the device
        assert adamw() == -2 and adamw(clip=e) == -2
        assert hnh.hnh_clip_coef_f64(a, b, 2, 1.0, None) == -2


def test_training_driver_entry_points_validate_without_a_gpu(hnh):
    out = C.c_void_p()
    lab = (C.c_int32 * 4)(0, 1, -1, 2)
    res = (C.c_double * 4)()
    assert hnh.hnhd_labels_create(None, lab, 4, 3, C.byref(out)) == -1 and b"null" in hnh.hnh_last_error_string()
    assert hnh.hnhd_labels_create(C.addressof(res), lab, 4, 3, None) == -1
    good = dict(lr=1e-3, b1=0.9, b2=0.999, eps=1e-8, wd=1e-2, mg=0.0)

    def create(**kw):
        a = dict(good, **kw)
        return hnh.hnhd_adamw_create(a["lr"], a["b1"], a["b2"], a["eps"], a["wd"], a["mg"], C.byref(out))

    for kw, what in ((dict(lr=-1e-3), b"lr"), (dict(lr=math.inf), b"lr"), (dict(lr=math.nan), b"lr"), (dict(b1=1.0), b"betas"),
                     (dict(b1=-0.1), b"betas"), (dict(b2=1.0), b"betas"), (dict(b2=math.nan), b"betas"), (dict(eps=0.0), b"eps"),
                     (dict(eps=-1e-8), b"eps"), (dict(wd=-1e-2), b"weight_decay"), (dict(wd=math.nan), b"weight_decay"),
                     (dict(mg=-1.0), b"max_grad_norm"), (dict(mg=math.nan), b"max_grad_norm")):
        assert create(**kw) == -1 and what in hnh.hnh_last_error_string(), kw
    assert hnh.hnhd_adamw_create(1e-3, 0.9, 0.999, 1e-8, 1e-2, 0.0, None) == -1
    assert create(mg=math.inf) == 0  # clipping at +inf never changes a gradient
    opt = C.c_void_p(out.value)
    assert hnh.hnhd_adamw_set_lr(opt, -1.0) == -1 and b"lr" in hnh.hnh_last_error_string()
    assert hnh.hnhd_adamw_set_lr(opt, math.nan) == -1
    assert hnh.hnhd_adamw_set_lr(opt, 0.5) == 0
    assert hnh.hnhd_adamw_set_lr(None, 0.5) == -1
    p = C.addressof(res)
    for args in ((None, p, opt), (p, None, opt), (p, p, None)):
        assert hnh.hnhd_gt_train_step(*args, 0.0, 0, res) == -1 and b"null" in hnh.hnh_last_error_string()
        assert hnh.hnhd_gat_train_step(*args, res) == -1 and b"null" in hnh.hnh_last_error_string()
    assert hnh.hnhd_gt_train_step(p, p, opt, 0.0, 0, None) == -1
    assert hnh.hnhd_gat_train_step(p, p, opt, None) == -1
    assert hnh.hnhd_gat_get_weight(None, 0, 0, p) == -1
    assert hnh.hnhd_gat_get_attention_vectors(None, 0, 0, p, p) == -1
    hnh.hnhd_adamw_destroy(opt)
    hnh.hnhd_labels_destroy(None)


def test_python_front_end_validates_training_arguments():
    from distributed_sddmm_b200 import driver as D
    with pytest.raises(ValueError, match="max_grad_norm"):
        D.AdamW(max_grad_norm=0.0)
    with pytest.raises(ValueError, match="max_grad_norm"):
        D.AdamW(max_grad_norm=-1.0)
    with pytest.raises(ValueError, match="max_grad_norm"):
        D.AdamW(max_grad_norm=math.nan)
    for kw in (dict(lr=-1.0), dict(betas=(1.0, 0.999)), dict(betas=(0.9, -0.5)), dict(eps=0.0), dict(weight_decay=-1.0)):
        with pytest.raises(RuntimeError, match="adamw_create failed"):
            D.AdamW(**kw)
    opt = D.AdamW()
    assert opt.lr == 1e-3
    opt.lr = 0.25
    assert opt.lr == 0.25
    with pytest.raises(RuntimeError, match="adamw_set_lr failed"):
        opt.lr = -1.0
    assert opt.lr == 0.25

    class Net:  # what NodeLabels reads of a model
        layers = [(4, 2, 2)]
        alg = type("A", (), {"h": None})()

        def buffer_shape(self, i):
            return (5, 4)

    with pytest.raises(ValueError, match="5 output rows"):
        D.NodeLabels(Net(), np.zeros(4, np.int64), 4)
    with pytest.raises(ValueError, match="integer"):
        D.NodeLabels(Net(), np.zeros(5), 4)
    with pytest.raises(ValueError, match="integer"):
        D.NodeLabels(Net(), np.zeros((5, 1), np.int32), 4)
    with pytest.raises(ValueError, match="int32"):
        D.NodeLabels(Net(), np.full(5, 1 << 40), 4)
    with pytest.raises(ValueError, match="num_classes"):
        D.NodeLabels(Net(), np.zeros(5, np.int32), 4.0)
    with pytest.raises(RuntimeError, match="labels_create failed"):
        D.NodeLabels(Net(), np.zeros(5, np.int32), 4)  # null algorithm handle
    gt = D.GraphTransformer.__new__(D.GraphTransformer)
    gt.h = None
    with pytest.raises(TypeError, match="NodeLabels"):
        gt.train_step(np.zeros(5), opt)
    labels = D.NodeLabels.__new__(D.NodeLabels)
    labels.h = None
    with pytest.raises(TypeError, match="AdamW"):
        gt.train_step(labels, None)
    with pytest.raises(ValueError, match="dropout"):
        gt.train_step(labels, opt, dropout=1.0)
    gat = D.GAT.__new__(D.GAT)
    gat.h = None
    with pytest.raises(TypeError, match="NodeLabels"):
        gat.train_step(None, opt)
