"""Relation-aware link prediction without a GPU: tests/distmult_oracle.py against PyG's example decoder built as an
nn.Module and against a per-triple loop, gradcheck of the loss, the op's conventions (entries that are no relation, one
H for both sides), and the Python-side argument checks of the driver classes, which refuse before any library call."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from distributed_sddmm_b200 import driver as D
from tests import distmult_oracle as dmo

SEED = 0xC0FFEE + 401


def _triples(rng, N, R, n):
    return rng.integers(0, N, n), rng.integers(0, N, n), rng.integers(0, R, n).astype(np.float64)


def test_oracle_matches_the_example_decoder():
    rng = np.random.default_rng(SEED)
    N, R, r = 40, 5, 8
    torch.manual_seed(0)
    dec = dmo.DistMultDecoder(R, r)
    z = torch.as_tensor(rng.standard_normal((N, r)))
    pos, neg = _triples(rng, N, R, 60), _triples(rng, N, R, 45)
    # the example's training loss, literally
    ei = lambda t: torch.stack([torch.as_tensor(t[0]), torch.as_tensor(t[1])])  # noqa: E731
    et = lambda t: torch.as_tensor(t[2].astype(np.int64))  # noqa: E731
    sp, sn = dec(z, ei(pos), et(pos)), dec(z, ei(neg), et(neg))
    want = F.binary_cross_entropy_with_logits(torch.cat([sp, sn]), torch.cat([torch.ones_like(sp), torch.zeros_like(sn)]))
    loss, correct, count, gp, gn = dmo.relational_loss(z, dec.rel_emb.detach(), pos, neg)
    assert abs(float(loss) - float(want.detach())) <= 1e-14 and count == 105
    assert np.abs(gp - sp.detach().numpy()).max() <= 1e-14 and np.abs(gn - sn.detach().numpy()).max() <= 1e-14
    assert correct == int((sp > 0).sum() + (sn <= 0).sum())
    # a per-triple loop
    D_ = dec.rel_emb.detach().numpy()
    Z = z.numpy()
    for (u, v, rho), s in zip(zip(*pos), gp):
        assert abs(sum(Z[u, k] * D_[int(rho), k] * Z[v, k] for k in range(r)) - s) <= 1e-13


def test_op_oracle_weights_sums_and_skips_non_relations():
    rng = np.random.default_rng(SEED + 1)
    N, R, r = 30, 3, 4
    H, H2, rel = rng.standard_normal((N, r)), rng.standard_normal((N, r)), rng.standard_normal((R, r))
    rows, cols, rels = _triples(rng, N, R, 50)
    bad = rels.copy()
    bad[:5] = [-1.0, 3.0, 0.5, np.nan, np.inf]
    l_all, c_all, s_all, a_all, b_all, d_all = dmo.op(H, H2, rel, rows, cols, rels, 1.0, 0.1)
    l_bad, c_bad, s_bad, *_ = dmo.op(H, H2, rel, rows, cols, bad, 1.0, 0.1)
    l_rest, c_rest, s_rest, a_rest, b_rest, d_rest = dmo.op(H, H2, rel, rows[5:], cols[5:], rels[5:], 1.0, 0.1)
    assert abs(l_bad - l_rest) <= 1e-13 and c_bad == c_rest and not s_bad[:5].any()
    assert np.abs(s_bad[5:] - s_rest).max() == 0
    # the gradients are inv_count times the sum's: a positive and a negative call add up to the mean over both
    lp, _, _, ap, _, dp = dmo.op(H, H, rel, rows, cols, rels, 1.0, 1 / 100, same=True)
    ln, _, _, an, _, dn = dmo.op(H, H, rel, cols, rows, rels, 0.0, 1 / 100, same=True)
    h, d = torch.as_tensor(H).requires_grad_(), torch.as_tensor(rel).requires_grad_()
    loss, *_ = dmo.relational_loss(h, d, (rows, cols, rels), (cols, rows, rels))
    loss.backward()
    assert abs((lp + ln) / 100 - float(loss)) <= 1e-13
    assert np.abs(ap + an - h.grad.numpy()).max() <= 1e-13 and np.abs(dp + dn - d.grad.numpy()).max() <= 1e-13


def test_gradcheck():
    rng = np.random.default_rng(SEED + 2)
    N, R, r = 9, 3, 4
    pos, neg = _triples(rng, N, R, 12), _triples(rng, N, R, 7)
    H = torch.as_tensor(rng.standard_normal((N, r))).requires_grad_()
    rel = torch.as_tensor(rng.standard_normal((R, r))).requires_grad_()
    assert torch.autograd.gradcheck(lambda h, d: dmo.relational_loss(h, d, pos, neg)[0], (H, rel))


class _Net:
    """Enough of a model for the argument checks that come before any library call."""
    layers = [(4, 4)]


def test_python_argument_checks():
    net = _Net()
    for bad in (0, -2, 1.5, True, "3"):
        with pytest.raises(ValueError, match="num_relations"):
            D.DistMultDecoder(net, bad)
    for bad in (1.5, True, None):
        with pytest.raises(ValueError, match="num_relations"):
            D.RelationalLinkTargets(net, object.__new__(D.Algorithm), object.__new__(D.Algorithm), bad)
    with pytest.raises(TypeError, match="alg_pos must be an Algorithm"):
        D.RelationalLinkTargets(net, None, object.__new__(D.Algorithm), 2)
    with pytest.raises(TypeError, match="alg_neg must be an Algorithm"):
        D.RelationalLinkTargets(net, object.__new__(D.Algorithm), "T", 2)
    m, dec = object.__new__(D.RGCN), object.__new__(D.DistMultDecoder)
    m.h = dec.h = None
    with pytest.raises(TypeError, match="decoder must be a DistMultDecoder"):
        m.relational_link_train_step(None, None, None)
    with pytest.raises(TypeError, match="targets must be a RelationalLinkTargets"):
        m.relational_link_evaluate(dec, object())
    alg = object.__new__(D.Algorithm)
    for kw, what in ((dict(num_relations=2.0), "num_relations"), (dict(num_relations=True), "num_relations"),
                     (dict(target="1"), "target"), (dict(inv_count=None), "inv_count")):
        args = dict(num_relations=2, target=1.0, inv_count=0.5)
        args.update(kw)
        with pytest.raises(ValueError, match=what):
            alg.distmult_loss(None, None, None, **args)
