"""Link prediction, CPU side: the fp64 oracle (tests/link_prediction_oracle.py) against F.binary_cross_entropy_with_logits
and finite differences, stable at |s| = 1000, and the new C and Python entry points refuse bad arguments without a GPU."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import link_prediction_oracle as lpo
from tests import training_oracle as tro
from tests.test_sparse_attention_bias import _pattern


def test_oracle_matches_torch_bce_and_finite_differences():
    rng = np.random.default_rng(1)
    N, r = 13, 4
    rows, cols = _pattern(rng, N, N, per_row=3)
    y = rng.choice([0.0, 1.0, 0.25], len(rows))
    H = rng.standard_normal((N, r))
    loss, correct, count, s, dA, dB = lpo.link_loss(H, H, rows, cols, y, same=True)
    st = torch.from_numpy((H[rows] * H[cols]).sum(1))
    assert math.isclose(loss, float(F.binary_cross_entropy_with_logits(st, torch.from_numpy(y))), rel_tol=1e-14)
    assert math.isclose(loss, float(lpo.bce_terms(st, torch.from_numpy(y)).mean()), rel_tol=1e-13)
    assert correct == int(((st > 0) == torch.from_numpy(y > 0.5)).sum()) and count == len(rows)
    assert dA is dB
    # dH_u = sum_v g_uv H_v + sum_w g_wu H_w
    g = (1 / (1 + np.exp(-s)) - y) / len(y)
    want = np.zeros_like(H)
    np.add.at(want, rows, g[:, None] * H[cols])
    np.add.at(want, cols, g[:, None] * H[rows])
    assert np.allclose(dA, want, rtol=1e-12, atol=1e-15)
    # separate H_A and H_B: each its own side
    H2 = rng.standard_normal((N, r))
    _, _, _, s2, gA, gB = lpo.link_loss(H, H2, rows, cols, y)
    g2 = (1 / (1 + np.exp(-s2)) - y) / len(y)
    wA, wB = np.zeros_like(H), np.zeros_like(H)
    np.add.at(wA, rows, g2[:, None] * H2[cols])
    np.add.at(wB, cols, g2[:, None] * H[rows])
    assert np.allclose(gA, wA, rtol=1e-12, atol=1e-15) and np.allclose(gB, wB, rtol=1e-12, atol=1e-15)


def test_oracle_is_stable_at_large_scores():
    """|s| = 1000: the loss is finite (s for a wrong sign, 0 for a right one), the gradient finite and of unit size."""
    H = np.array([[10.0, 0.0], [100.0, 0.0], [-100.0, 0.0]])  # s(0, 1) = 1000, s(0, 2) = -1000
    rows, cols = np.array([0, 0, 0, 0]), np.array([1, 1, 2, 2])
    y = np.array([1.0, 0.0, 1.0, 0.0])
    loss, correct, count, s, dH, _ = lpo.link_loss(H, H, rows, cols, y, same=True)
    assert np.array_equal(s, [1000.0, 1000.0, -1000.0, -1000.0])
    assert math.isclose(loss, (0 + 1000 + 1000 + 0) / 4, rel_tol=1e-15) and correct == 2 and count == 4
    assert np.isfinite(dH).all() and np.abs(dH).max() <= 100
    t = lpo.bce_terms(torch.from_numpy(s), torch.from_numpy(y))
    assert torch.isfinite(t).all()


def test_oracle_without_entries_is_zero():
    H = np.ones((4, 3))
    loss, correct, count, s, dH, _ = lpo.link_loss(H, H, [], [], [], same=True)
    assert (loss, correct, count) == (0.0, 0, 0) and not dH.any()


def test_link_training_oracle_uses_the_node_classification_models():
    """train_gt with the link loss equals a hand-written loop over the same forward (gto.model_torch)."""
    from tests import graph_transformer_block_oracle as gbo
    from tests import graph_transformer_oracle as gto
    rng = np.random.default_rng(4)
    N, layers = 11, [(3, 2, 2)]
    rows, cols = _pattern(rng, N, N, per_row=2)
    tr, tc = _pattern(rng, N, N, per_row=2)
    y = rng.choice([0.0, 1.0], len(tr))
    params = gbo.random_params(layers, 0, False, 0, rng)
    X = rng.standard_normal((N, 3))
    res, trained = lpo.train_gt(rows, cols, N, layers, params, X, (tr, tc, y), 2, lr=0.05)
    tp = [{k: gto._t(v).clone().requires_grad_() for k, v in P.items()} for P in params]
    leaves = [v for P in tp for v in P.values()]
    opt = torch.optim.AdamW(leaves, lr=0.05, foreach=False)
    for t in range(2):
        opt.zero_grad()
        H = gto.model_torch(rows, cols, N, layers, tp, gto._t(X))
        s = (H[torch.as_tensor(tr)] * H[torch.as_tensor(tc)]).sum(1)
        loss = F.binary_cross_entropy_with_logits(s, torch.from_numpy(y))
        loss.backward()
        assert math.isclose(float(loss.detach()), res[t][0], rel_tol=1e-14) and res[t][2] == len(y)
        opt.step()
    for k, v in tp[0].items():
        assert np.allclose(v.detach().numpy(), trained[0][k], rtol=1e-13, atol=1e-15), k
    assert tro.train is not lpo.link_train_step  # the swap is undone


def test_auc():
    assert lpo.auc([0.1, 0.2, 0.9, 0.8], [0, 0, 1, 1]) == 1.0
    assert lpo.auc([0.9, 0.8, 0.1, 0.2], [0, 0, 1, 1]) == 0.0
    assert lpo.auc([0.5, 0.5, 0.5, 0.5], [0, 1, 0, 1]) == 0.5


def test_link_kernels_validate_without_a_gpu(hnh):
    bufs = [(C.c_double * 64)() for _ in range(8)]
    rs, ci, t, x, y, dx, st, sc = (C.addressof(b) for b in bufs)

    def bce(rs=rs, ci=ci, t=t, rows=4, nnz=4, x=x, ldx=4, y=y, ldy=4, r=4, inv=0.25, dx=dx, lddx=4, st=st, lds=2, sc=sc):
        return hnh.hnh_link_bce_f64(rs, ci, t, rows, nnz, x, ldx, y, ldy, r, inv, dx, lddx, st, lds, sc, None)

    assert bce(rows=-1) == -1 and b"negative" in hnh.hnh_last_error_string()
    assert bce(r=0) == -1 and b"r must be positive" in hnh.hnh_last_error_string()
    for kw in (dict(ldx=3), dict(ldy=3), dict(lddx=3)):
        assert bce(**kw) == -1 and b"leading dimension" in hnh.hnh_last_error_string(), kw
    assert bce(lds=1) == -1 and b"stats" in hnh.hnh_last_error_string()
    for bad in (-1.0, math.nan, math.inf):
        assert bce(inv=bad) == -1 and b"inv_count" in hnh.hnh_last_error_string()
    for k in ("rs", "ci", "t", "x", "y"):
        assert bce(**{k: None}) == -1 and b"null" in hnh.hnh_last_error_string(), k
    assert bce(dx=x) == -1 and b"may not be an input" in hnh.hnh_last_error_string()
    assert bce(sc=t) == -1 and b"may not be an input" in hnh.hnh_last_error_string()
    assert bce(st=dx) == -1 and b"distinct" in hnh.hnh_last_error_string()
    assert bce(rows=0) == 0 and bce(nnz=0, rs=None) == 0  # empty blocks are a no-op
    assert hnh.hnh_link_target_check_f64(st, t, -1, None) == -1
    assert hnh.hnh_link_target_check_f64(None, t, 4, None) == -1 and hnh.hnh_link_target_check_f64(st, None, 4, None) == -1
    assert hnh.hnh_link_target_check_f64(st, None, 0, None) == 0
    assert hnh.hnh_pair_sums_workspace_bytes(-1) == -1 and hnh.hnh_pair_sums_workspace_bytes(1000) >= 16
    assert hnh.hnh_pair_sums_f64(None, st, 4, sc, 1 << 10, None) == -1
    assert hnh.hnh_pair_sums_f64(st, st, 4, None, 0, None) == -1 and b"workspace" in hnh.hnh_last_error_string()
    if not torch.cuda.is_available():  # no CPU fallback: compute fails with HNH_E_CUDA
        assert bce() == -2
        assert hnh.hnh_link_target_check_f64(st, t, 4, None) == -2


def test_link_driver_entry_points_validate_without_a_gpu(hnh):
    out = C.c_void_p()
    res = (C.c_double * 4)()
    p = C.addressof(res)
    assert hnh.hnhd_alg_link_loss(None, p, p, None, None, None, res) == -1 and b"null" in hnh.hnh_last_error_string()
    assert hnh.hnhd_alg_link_loss(p, None, p, None, None, None, res) == -1
    assert hnh.hnhd_alg_link_loss(p, p, p, None, None, None, None) == -1
    assert hnh.hnhd_link_targets_create(None, p, C.byref(out)) == -1 and b"null" in hnh.hnh_last_error_string()
    assert hnh.hnhd_link_targets_create(p, None, C.byref(out)) == -1
    assert hnh.hnhd_link_targets_create(p, p, None) == -1
    for args in ((None, p, p), (p, None, p), (p, p, None)):
        assert hnh.hnhd_gt_link_train_step(*args, 0.0, 0, res) == -1 and b"null" in hnh.hnh_last_error_string()
        assert hnh.hnhd_gat_link_train_step(*args, res) == -1 and b"null" in hnh.hnh_last_error_string()
    assert hnh.hnhd_gt_link_train_step(p, p, p, 0.0, 0, None) == -1
    assert hnh.hnhd_gt_link_evaluate(None, p, None, res) == -1 and hnh.hnhd_gat_link_evaluate(p, None, None, res) == -1
    assert hnh.hnhd_gt_link_evaluate(p, p, None, None) == -1
    hnh.hnhd_link_targets_destroy(None)


def test_python_front_end_validates_link_arguments():
    from distributed_sddmm_b200 import driver as D
    alg = D.Algorithm.__new__(D.Algorithm)
    alg.h = None
    with pytest.raises(TypeError, match="H_A must be a Dense"):
        alg.link_loss(np.zeros((2, 2)), None)
    dense = D.Dense.__new__(D.Dense)
    dense.h = None
    with pytest.raises(TypeError, match="dH_B must be a Dense"):
        alg.link_loss(dense, dense, None, np.zeros(2))
    with pytest.raises(TypeError, match="scores must be a Vec"):
        alg.link_loss(dense, dense, scores=[0.0])
    with pytest.raises(RuntimeError, match="link_loss failed"):
        alg.link_loss(dense, dense)  # null algorithm handle

    class Net:
        alg = type("A", (), {"h": None})()

    with pytest.raises(TypeError, match="alg_T must be an Algorithm"):
        D.LinkTargets(Net(), None)
    with pytest.raises(RuntimeError, match="link_targets_create failed"):
        D.LinkTargets(Net(), alg)
    opt = D.AdamW()
    for net in (D.GraphTransformer.__new__(D.GraphTransformer), D.GAT.__new__(D.GAT)):
        net.h = None
        with pytest.raises(TypeError, match="LinkTargets"):
            net.link_train_step(None, opt)
        with pytest.raises(TypeError, match="LinkTargets"):
            net.link_evaluate(object())
    targets = D.LinkTargets.__new__(D.LinkTargets)
    targets.h = None
    gt = D.GraphTransformer.__new__(D.GraphTransformer)
    gt.h = None
    with pytest.raises(TypeError, match="AdamW"):
        gt.link_train_step(targets, None)
    with pytest.raises(ValueError, match="dropout"):
        gt.link_train_step(targets, opt, dropout=1.0)
