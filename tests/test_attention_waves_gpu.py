"""The edge softmax and additive-attention kernels past one resident wave, and the edge softmax on masked (-inf) scores.

Those kernels cap their grids at GRID_PER_SM CTAs of THREADS threads per SM.  The reductions run one warp per plan
piece, then one warp per row; the elementwise kernels one thread per entry.  Each case is sized from the device's SM
count so that every warp or thread runs at least WAVES grid-stride iterations, with rows of 1023 to 2049 entries
(one and two pieces) and empty rows among them.

-inf is the usual mark of a masked edge: the expected result is torch.softmax over the row's entries, which gives 0
to a masked entry and NaN to every entry of a row that is masked throughout."""
import numpy as np
import pytest

from distributed_sddmm_b200 import driver as D
from tests import gat_softmax_oracle as gso

pytestmark = pytest.mark.gpu

WAVES = 3
GRID_PER_SM = 16  # kCtasPerSm in csrc/edge_softmax.cu and csrc/gat_additive.cu
THREADS = 256     # kBlock (csrc/launch.h)
PIECE = 1024      # kPiece: entries of a row one warp reduces
ALPHA = 0.2


def bounds(sms):
    """Work that makes every warp (one per piece / row) and every thread (one per entry) of the largest grid run WAVES
    iterations."""
    threads = WAVES * GRID_PER_SM * sms * THREADS
    return dict(warps=threads // 32, threads=threads)


def softmax_keys(sms, seed=51):
    """Row keys in shuffled order: more non-empty rows (so more pieces) than the warp bound, more entries than the
    thread bound, every tenth row empty, rows of 1023, 1024, 1025, 2048, 2049 and 5000 entries early and late."""
    b = bounds(sms)
    M = -(-b["warps"] * 10 // 9) + 64
    rng = np.random.default_rng(seed)
    mean = -(-b["threads"] * 10 // (9 * M)) + 1
    lens = rng.integers(1, 2 * mean, M)
    lens[::10] = 0
    special = [1023, 1024, 1025, 2048, 2049, 5000]
    lens[1:1 + len(special)] = special
    lens[M - 1 - len(special):M - 1] = special
    keys = np.repeat(np.arange(M), lens)
    rng.shuffle(keys)
    return keys, M


@pytest.fixture(scope="module")
def world():
    D.world_init("self")
    yield
    D.world_finalize()


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _close(got, want, rtol=1e-13):
    assert got.shape == want.shape
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), np.flatnonzero(np.isnan(got) != nan)[:5]
    g, w = got[~nan], want[~nan]
    err = np.abs(g - w).max() if len(w) else 0.0
    assert err <= rtol * max(np.abs(w).max(), 1e-300), err


# ---- edge softmax past one wave ---------------------------------------------------------------------------------
def test_edge_softmax_kernels_past_one_wave(world, sms):
    import torch
    from distributed_sddmm_b200 import lib
    from tests.test_edge_softmax_gpu import _backward, _plan, _softmax
    L = lib()
    dev = torch.device("cuda:0")
    keys, M = softmax_keys(sms)
    b = bounds(sms)
    pl = _plan(L, torch, dev, keys, M)
    lens = np.bincount(keys, minlength=M)
    assert pl["P"] == int(np.sum(-(-lens // PIECE)))
    assert pl["P"] >= b["warps"] and M >= b["warps"] and len(keys) >= b["threads"], (pl["P"], M, len(keys), b)
    perm = pl["perm"].cpu().numpy()
    assert np.array_equal(perm, np.argsort(keys, kind="stable"))
    rng = np.random.default_rng(52)
    x_np = rng.uniform(-300, 300, len(keys))
    x = torch.from_numpy(x_np).to(dev)
    a, rm, rsum = _softmax(L, torch, dev, pl, x)
    got = a.cpu().numpy()
    want = gso.edge_softmax_np(x_np, keys, M)
    assert np.isfinite(got).all()
    assert np.abs(got - want).max() <= 1e-13 * np.abs(want).max()
    empty = lens == 0
    assert np.all(rm.cpu().numpy()[empty] == -np.inf) and np.all(rsum.cpu().numpy()[empty] == 0)
    m = np.full(M, -np.inf)
    np.maximum.at(m, keys, x_np)
    assert np.array_equal(rm.cpu().numpy(), m)
    a2, rm2, rsum2 = _softmax(L, torch, dev, pl, x)
    assert torch.equal(a, a2) and torch.equal(rm, rm2) and torch.equal(rsum, rsum2)
    # backward: the row dot, then the elementwise apply
    g_np = rng.uniform(-1, 1, len(keys))
    g = torch.from_numpy(g_np).to(dev)
    dx, rd = _backward(L, torch, dev, pl, a, g)
    want_dx = gso.edge_softmax_backward_np(got, g_np, keys, M)
    assert np.abs(dx.cpu().numpy() - want_dx).max() <= 1e-13 * np.abs(want_dx).max()
    abs_sum = np.bincount(keys, weights=np.abs(got * g_np), minlength=M)
    assert np.all(np.abs(rd.cpu().numpy() - np.bincount(keys, weights=got * g_np, minlength=M)) <= 1e-12 * abs_sum)
    assert np.all(rd.cpu().numpy()[empty] == 0)
    dx2, rd2 = _backward(L, torch, dev, pl, a, g)
    assert torch.equal(dx, dx2) and torch.equal(rd, rd2)
    # row sums over the plan
    sums = []
    for _ in range(2):
        ps = torch.full((max(pl["P"], 1),), float("nan"), dtype=torch.float64, device=dev)
        out = torch.full((M,), float("nan"), dtype=torch.float64, device=dev)
        D.check(L.hnh_edge_sum_f64(g.data_ptr(), pl["perm"].data_ptr(), pl["rs"].data_ptr(), pl["pf"].data_ptr(), pl["pr"].data_ptr(),
                                   M, pl["P"], ps.data_ptr(), out.data_ptr(), pl["st"]))
        torch.cuda.synchronize()
        sums.append(out.cpu().numpy())
    want_s = np.bincount(keys, weights=g_np, minlength=M)
    assert np.all(np.abs(sums[0] - want_s) <= 1e-12 * np.bincount(keys, weights=np.abs(g_np), minlength=M))
    assert np.all(sums[0][empty] == 0) and np.array_equal(sums[0], sums[1])


# ---- additive-attention kernels past one wave -------------------------------------------------------------------
@pytest.mark.parametrize("d,shift", [(64, 0), (7, 0), (12, 1)], ids=["paired", "odd_d", "offset"])
def test_node_scalars_and_rank2_update_past_one_wave(world, sms, d, shift):
    """One warp per row: paired 16-byte loads (even d, aligned), scalar loads (odd d, or an 8-byte offset)."""
    import torch
    from distributed_sddmm_b200 import lib
    L = lib()
    dev = torch.device("cuda:0")
    st = torch.cuda.current_stream().cuda_stream
    n = bounds(sms)["warps"] + 13
    assert n >= bounds(sms)["warps"]
    rng = np.random.default_rng(53 + d)
    f64 = dict(dtype=torch.float64, device=dev)
    P_np = rng.uniform(-1, 1, (n, d))
    a1_np, a2_np = rng.uniform(-1, 1, d), rng.uniform(-1, 1, d)
    P = torch.zeros(n * d + shift, **f64)
    P[shift:] = torch.from_numpy(P_np.ravel())
    a = torch.zeros(2 * d + 2 * shift, **f64)
    a[shift:shift + d] = torch.from_numpy(a1_np)
    a[d + 2 * shift:] = torch.from_numpy(a2_np)
    a1p, a2p = a.data_ptr() + 8 * shift, a.data_ptr() + 8 * (d + 2 * shift)
    res = []
    for _ in range(2):
        s, t = torch.full((n,), float("nan"), **f64), torch.full((n,), float("nan"), **f64)
        D.check(L.hnh_gat_node_scalars_f64(s.data_ptr(), t.data_ptr(), P.data_ptr() + 8 * shift, a1p, a2p, n, d, st))
        torch.cuda.synchronize()
        res.append((s.cpu().numpy(), t.cpu().numpy()))
    s_np, t_np = res[0]
    assert np.abs(s_np - P_np @ a1_np).max() <= 1e-13 * np.abs(P_np @ a1_np).max()
    assert np.abs(t_np - P_np @ a2_np).max() <= 1e-13 * np.abs(P_np @ a2_np).max()
    assert np.array_equal(res[0][0], res[1][0]) and np.array_equal(res[0][1], res[1][1])
    ds_np, dt_np = rng.uniform(-1, 1, n), rng.uniform(-1, 1, n)
    ds, dt = torch.from_numpy(ds_np).to(dev), torch.from_numpy(dt_np).to(dev)
    D.check(L.hnh_gat_rank2_update_f64(P.data_ptr() + 8 * shift, ds.data_ptr(), dt.data_ptr(), a1p, a2p, n, d, st))
    torch.cuda.synchronize()
    want = P_np + np.outer(ds_np, a1_np) + np.outer(dt_np, a2_np)
    assert np.abs(P[shift:].cpu().numpy().reshape(n, d) - want).max() <= 1e-14 * np.abs(want).max()
    if shift:
        assert P[0].item() == 0.0  # the word before the offset rows is left alone


def test_edge_scores_past_one_wave(world, sms):
    import torch
    from distributed_sddmm_b200 import lib
    L = lib()
    dev = torch.device("cuda:0")
    st = torch.cuda.current_stream().cuda_stream
    n = bounds(sms)["threads"] + 77
    rng = np.random.default_rng(57)
    nr, nc = 70001, 65003
    rk, ck = rng.integers(0, nr, n), rng.integers(0, nc, n)
    s_np, t_np = rng.uniform(-1, 1, nr), rng.uniform(-1, 1, nc)
    s_np[0] = -t_np[0]
    rk[::9], ck[::9] = 0, 0  # s + t == 0 exactly: LeakyReLU'(0) = alpha
    x = s_np[rk] + t_np[ck]
    rkd, ckd = (torch.from_numpy(k.astype(np.int32)).to(dev) for k in (rk, ck))
    s, t = torch.from_numpy(s_np).to(dev), torch.from_numpy(t_np).to(dev)
    for derivative, want in ((0, np.maximum(x, 0.0) + np.minimum(x, 0.0) * ALPHA), (1, np.where(x > 0, 1.0, ALPHA))):
        out = torch.full((n,), float("nan"), dtype=torch.float64, device=dev)
        D.check(L.hnh_gat_edge_scores_f64(out.data_ptr(), s.data_ptr(), t.data_ptr(), rkd.data_ptr(), ckd.data_ptr(), n, ALPHA,
                                          derivative, st))
        torch.cuda.synchronize()
        assert np.array_equal(out.cpu().numpy(), want), derivative


# ---- masked (-inf) scores -----------------------------------------------------------------------------------------
def _torch_rows(x, keys, M, g=None):
    """Per row, torch.softmax over the row's entries (and, with g, the gradient of <g, softmax> by autograd)."""
    import torch
    alpha, dx = np.empty_like(x), np.empty_like(x)
    for u in range(M):
        idx = np.flatnonzero(keys == u)
        if not len(idx):
            continue
        xt = torch.tensor(x[idx], requires_grad=True)
        y = torch.softmax(xt, 0)
        alpha[idx] = y.detach().numpy()
        if g is not None:
            y.backward(torch.from_numpy(g[idx]))
            dx[idx] = xt.grad.numpy()
    return alpha, dx


def _masked_rows():
    """(keys, M, lens, mask in perm order per row): rows longer than 32 entries with -inf where a lane starts."""
    spec = [  # (length, positions in the row's perm order that are -inf)
        (64, [3]),
        (100, list(range(32))),
        (50, list(range(50))),               # masked throughout
        (2000, list(range(1024))),           # a whole piece masked
        (1100, [0] + list(range(1024, 1056))),  # the lanes' first entries of the second piece
        (40, list(range(0, 40, 2))),
        (5, [0]),
        (0, []),
        (33, [32]),
        (70, list(range(1, 70))),            # one finite entry, at perm position 0
    ]
    return spec


def test_edge_softmax_masked_scores(world):
    import torch
    from distributed_sddmm_b200 import lib
    from tests.test_edge_softmax_gpu import _backward, _plan, _softmax
    L = lib()
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(59)
    spec = _masked_rows()
    M = len(spec)
    keys = np.repeat(np.arange(M), [n for n, _ in spec])
    rng.shuffle(keys)
    perm = np.argsort(keys, kind="stable")
    rs = np.searchsorted(keys[perm], np.arange(M + 1))
    x_np = rng.uniform(-30, 30, len(keys))
    for u, (_, masked) in enumerate(spec):
        x_np[perm[rs[u] + np.array(masked, np.int64)]] = -np.inf
    g_np = rng.uniform(-1, 1, len(keys))
    want, want_dx = _torch_rows(x_np, keys, M, g_np)
    pl = _plan(L, torch, dev, keys, M)
    assert np.array_equal(pl["perm"].cpu().numpy(), perm)
    x = torch.from_numpy(x_np).to(dev)
    a, rm, rsum = _softmax(L, torch, dev, pl, x)
    got = a.cpu().numpy()
    _close(got, want)
    full = np.array([len(m) == n and n > 0 for n, m in spec])
    assert np.all(np.isnan(got[full[keys]])) and not np.isnan(got[~full[keys]]).any()
    assert np.all(got[np.isneginf(x_np) & ~full[keys]] == 0.0)
    # row statistics: a row masked throughout is (-inf, 0) like an empty row; every other row's sum is finite
    rm_np, rs_np = rm.cpu().numpy(), rsum.cpu().numpy()
    assert np.all(rm_np[full] == -np.inf) and np.all(rs_np[full] == 0)
    assert np.all(np.isfinite(rs_np)) and np.all(rs_np[~full & (np.bincount(keys, minlength=M) > 0)] >= 1)
    dx, _ = _backward(L, torch, dev, pl, a, torch.from_numpy(g_np).to(dev))
    _close(dx.cpu().numpy(), want_dx)


@pytest.mark.parametrize("name", ["15d_fusion2", "15d_fusion1"])
def test_p1_edge_softmax_masked_scores(world, name):
    """Algorithm.edge_softmax / edge_softmax_backward at p = 1 on scores with masked entries, in both value orders."""
    from tests.test_edge_softmax_gpu import _entry_coords, _score
    N = 256
    rng = np.random.default_rng(61)
    r = rng.integers(0, N, 1500)
    c = rng.integers(0, N, 1500)
    for u, n in ((3, 40), (77, 64), (200, 50), (255, 90)):  # rows longer than 32 entries
        r = np.concatenate([r, np.full(n, u)])
        c = np.concatenate([c, rng.choice(N, n, replace=False)])
    key = np.unique(r * N + c)
    r, c = key // N, key % N
    S = D.SpmatLocal.from_tuples(N, N, r, c, np.ones(len(r)))
    alg = D.Algorithm(name, S, 8, 1)
    for mode in ("A", "B"):
        er, ec = _entry_coords(alg, name, mode)
        x = _score(er, ec)
        x[(er == 3) & (ec != ec[er == 3].max())] = -np.inf   # all but one entry
        x[(er == 77) & (ec % 2 == 0)] = -np.inf
        x[er == 200] = -np.inf                              # masked throughout
        x[(er == 255) & (ec < 128)] = -np.inf
        x[(er < 40) & (ec % 5 == 0)] = -np.inf
        g = np.cos(0.5 * er - 0.3 * ec)
        want, want_dx = _torch_rows(x, er, N, g)
        like = alg.like_S_values if mode == "A" else alg.like_ST_values
        v = like(0.0)
        v.from_host(x)
        alg.edge_softmax(v, mode)
        a = v.to_host()
        _close(a, want)
        assert np.isnan(a[er == 200]).all() and np.all(a[np.isneginf(x) & (er != 200)] == 0)
        gv = like(0.0)
        gv.from_host(g)
        alg.edge_softmax_backward(v, gv, mode)
        _close(gv.to_host(), want_dx)
