"""The transformer block's kernels alone on the GPU: hnh_layer_norm_f64 and hnh_layer_norm_backward_f64 against torch's
fp64 LayerNorm and its autograd, and hnh_row_bias_relu_f64 against numpy.  Past one resident wave (50 000 rows); r = 1,
odd r, r on every register-row width up to 1536 and wider than the register paths; rows shifted by one double
(misaligned: the scalar path); with and without the residual; rows with a mean of 1e8 and a standard deviation of 1
(where E[x^2] - E[x]^2 loses every digit) and constant rows (var = 0, rstd = 1 / sqrt(eps)); dgamma and dbeta
bit-identical over repeats; the add-to flag."""
import numpy as np
import pytest
import torch

from distributed_sddmm_b200 import check, lib

pytestmark = pytest.mark.gpu


def rel_err(got, ref, floor=1e-300):
    return np.abs(got - ref).max() / max(np.abs(ref).max(), floor)


class Dev:
    """Device copies of host arrays at an offset of `shift` doubles (shift = 1: rows not 16-byte aligned)."""

    def __init__(self, shift):
        self.shift = shift
        self.keep = []

    def __call__(self, x):
        x = np.asarray(x, np.float64)
        t = torch.zeros(x.size + 2, dtype=torch.float64, device="cuda")
        t[self.shift:self.shift + x.size] = torch.from_numpy(x.reshape(-1))
        self.keep.append((t, x.shape))
        return t.data_ptr() + 8 * self.shift

    def host(self, ptr):
        torch.cuda.synchronize()
        for t, shape in self.keep:
            if t.data_ptr() + 8 * self.shift == ptr:
                return t[self.shift:self.shift + int(np.prod(shape))].cpu().numpy().reshape(shape)
        raise KeyError(ptr)


def reference(X, Res, gamma, beta, G, eps):
    """torch fp64 LayerNorm of X + Res: (Y, mean, rstd, dX, dgamma, dbeta) for the output gradient G."""
    x = torch.from_numpy(X + (Res if Res is not None else 0)).requires_grad_()
    g, b = (torch.from_numpy(v).requires_grad_() for v in (gamma, beta))
    y = torch.nn.functional.layer_norm(x, (X.shape[1],), g, b, eps)
    y.backward(torch.from_numpy(G))
    xd = x.detach().numpy()
    mean = xd.mean(1)
    var = ((xd - mean[:, None]) ** 2).mean(1)
    return y.detach().numpy(), mean, 1 / np.sqrt(var + eps), x.grad.numpy(), g.grad.numpy(), b.grad.numpy()


def run(n, r, shift, res, rng, eps=1e-5, X=None, tol=1e-12):
    L = lib()
    st = torch.cuda.current_stream().cuda_stream
    if X is None:
        X = rng.uniform(-2, 3, (n, r))
    Res = rng.uniform(-1, 1, (n, r)) if res else None
    gamma, beta, G = rng.uniform(0.5, 1.5, r), rng.uniform(-1, 1, r), rng.uniform(-1, 1, (n, r))
    d = Dev(shift)
    pX, pR, pg, pb, pG = d(X), d(Res) if res else None, d(gamma), d(beta), d(G)
    pY, pS = d(np.full((n, r), np.nan)), d(np.full((n, 2), np.nan))
    check(L.hnh_layer_norm_f64(pY, pS, pX, pR, pg, pb, n, r, eps, st), "layer_norm")
    Yw, mean, rstd, dXw, dgw, dbw = reference(X, Res, gamma, beta, G, eps)
    assert rel_err(d.host(pY), Yw) < tol, (n, r, shift, res)
    stats = d.host(pS)
    assert rel_err(stats[:, 0], mean) < 1e-13 and rel_err(stats[:, 1], rstd) < tol
    ws_bytes = L.hnh_layer_norm_backward_workspace_bytes(n, r)
    ws = torch.full((max(ws_bytes, 8) // 8,), np.nan, dtype=torch.float64, device="cuda")
    prev = rng.uniform(-1, 1, (n, r))
    pdX, pdg, pdb = d(prev), d(np.full(r, np.nan)), d(np.full(r, np.nan))
    dgs = []
    for acc in (1, 0, 0):  # add-to first (dX holds `prev`), then overwrite twice
        check(L.hnh_layer_norm_backward_f64(pdX, pdg, pdb, pG, pX, pR, pS, pg, n, r, acc, ws.data_ptr(), ws_bytes, st),
              "layer_norm_backward")
        if acc:
            assert rel_err(d.host(pdX), prev + dXw, 1.0) < tol
        dgs.append((d.host(pdg).copy(), d.host(pdb).copy()))
    assert rel_err(d.host(pdX), dXw, 1.0) < tol  # against at least 1: dX is 0 up to rounding for r = 1
    # dgamma against at least 1 too: for r = 1, xh = 0 and dgamma is 0 up to rounding
    assert rel_err(dgs[0][0], dgw, 1.0) < max(tol, 1e-11) and rel_err(dgs[0][1], dbw) < 1e-11
    assert all(np.array_equal(a[0], dgs[0][0]) and np.array_equal(a[1], dgs[0][1]) for a in dgs)
    return d.host(pY), stats


@pytest.mark.parametrize("r", [1, 7, 64, 128, 250, 512, 768, 1024, 1536, 1538, 2047])
def test_layer_norm_widths(r):
    """Every register-row width (r <= 64 kN), odd ones, past the backward's (1024) and the forward's (1536) register
    rows; n past one resident wave for the narrow rows."""
    rng = np.random.default_rng(r)
    n = 50000 if r <= 128 else 4000
    for shift in (0, 1):
        for res in (False, True):
            run(n, r, shift, res, rng)


def test_layer_norm_past_one_wave_wide():
    run(50000, 1024, 0, True, np.random.default_rng(3))


@pytest.mark.parametrize("r", [64, 1024, 2000, 33])
def test_layer_norm_large_mean(r):
    """Rows of mean 1e8 and standard deviation 1: a one-pass variance (E[x^2] - E[x]^2) cancels to noise here."""
    rng = np.random.default_rng(r + 1)
    n = 2000
    X = 1e8 + rng.standard_normal((n, r))
    for shift in (0, 1):
        Y, stats = run(n, r, shift, False, rng, X=X, tol=1e-6)
        sd = X.std(1)
        assert np.allclose(stats[:, 1], 1 / np.sqrt(sd ** 2 + 1e-5), rtol=1e-6)


@pytest.mark.parametrize("r", [1, 6, 1024, 1600])
def test_layer_norm_constant_rows(r):
    """var = 0: Y = beta, rstd = 1 / sqrt(eps) exactly, dX = rstd (g - mean(g))."""
    rng = np.random.default_rng(r + 2)
    n = 300
    X = np.repeat(rng.uniform(-5, 5, (n, 1)), r, axis=1)
    eps = 1e-3
    Y, stats = run(n, r, 0, False, rng, eps=eps, X=X)
    assert np.array_equal(stats[:, 1], np.full(n, 1 / np.sqrt(eps)))
    assert np.allclose(stats[:, 0], X[:, 0], rtol=1e-14, atol=0) and np.allclose(Y, np.broadcast_to(Y[:1], Y.shape), atol=1e-12)


@pytest.mark.parametrize("r", [6, 7])
def test_row_bias_relu(r):
    L = lib()
    st = torch.cuda.current_stream().cuda_stream
    rng = np.random.default_rng(r)
    n = 50000
    A, b = rng.uniform(-1, 1, (n, r)), rng.uniform(-1, 1, r)
    for shift in (0, 1):
        d = Dev(shift)
        pA, pb, pZ = d(A), d(b), d(np.full((n, r), np.nan))
        check(L.hnh_row_bias_relu_f64(pZ, pA, pb, n, r, st), "row_bias_relu")
        assert np.array_equal(d.host(pZ), np.maximum(A + b, 0.0))
