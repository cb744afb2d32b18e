"""The SDDMM / SpMM / fused engine past one resident wave: the row-length fixture, the exact reference and the checks
shared by tests/test_kernel_waves_gpu.py (in process) and its child processes (`python -m tests.kernel_waves_worker
<group>`, for the paths that HNH_SPLIT_MAX_R and HNH_TMA select: the library reads them once per process).

Every kernel walks its work with a grid-stride loop, and grid_for (csrc/launch.h) caps the grid at the CTAs resident
at once, at most 8 per SM for 256-thread CTAs.  Each case is sized from its kernel's work unit per CTA so that every
CTA runs at least WAVES iterations, which is where the later iterations, the TMA next-tile prefetch and the second
mbarrier phase run.

Operands are small nonzero integers and the scale factors powers of two, with every partial sum far below 2^53, so
every result is exact in fp64 whatever the summation order: each output must be bit-equal to the numpy / scipy
reference.  Outputs that a flag says are overwritten start as NaN.

Run as a program, the worker checks one group and exits 1 after printing the first mismatch."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

# ---- the launchers' constants (csrc/launch.h, row_gather.cuh, c_abi.cu; tests/test_kernel_waves.py reads them back) --
BLOCK = 256                # kBlock: threads per CTA
CTAS_PER_SM = 2048 // BLOCK  # the most 256-thread CTAs an SM holds, so the most grid_for ever launches per SM
WAVES = 3                  # grid-stride iterations every CTA must run at least
SPLIT = {4: (2, 8, 4), 8: (4, 8, 4), 16: (8, 4, 4), 32: (16, 2, 4)}  # HNH_DISPATCH_SPLIT: r -> (GK, GN, UN)
ROW_G = {4: 2, 8: 4, 16: 8, 32: 16, 64: 32, 128: 32, 256: 32}      # HNH_DISPATCH_R: r -> G lanes per row
TABLE = sorted(ROW_G)
TILE = 8                   # rows per CTA iteration of the TMA kernels and the one-warp-per-row generic kernels
COO_UNIT = BLOCK           # nonzeros per CTA iteration of sddmm_coo_kernel: (256 / G) groups of G

FORCE_GENERIC, FORCE_DIRECT, BETA0, BETA0_VALUES, BETA0_OUT, TMA_STAGE, TMA_WARP, SCALE_VALUES = 1, 2, 4, 16, 32, 64, 128, 256
LONG_ROWS = (20000, 1000, 4099, 20000)  # placed early, in the middle and late
EMPTY_RUN = 24             # consecutive empty rows from a tile boundary: whole TMA tiles without work
OPERAND = np.array([-3.0, -2.0, -1.0, 1.0, 2.0, 3.0])
SCALES = np.array([-4.0, -2.0, -1.0, -0.5, -0.25, 0.25, 0.5, 1.0, 2.0, 4.0])
VMAX, SMAX = 4.0, 4.0      # |initial values|, |scale|


def units_per_cta(path, r):
    """Rows (entries for "coo") that one CTA handles per grid-stride iteration on `path`."""
    if path == "split":
        gk, gn, _ = SPLIT[r]
        return BLOCK // (gk * gn)
    if path == "row":
        return BLOCK // ROW_G[r]
    if path in ("tma", "generic"):
        return TILE
    if path == "coo":
        return COO_UNIT
    raise ValueError(path)


def wave_bound(units, sms):
    """Work units that make every CTA of the largest possible grid run WAVES iterations."""
    return WAVES * CTAS_PER_SM * sms * units


def rows_for(units, sms):
    """The first row count past the wave bound that is not a multiple of 8 (the last TMA tile is partial)."""
    m = wave_bound(units, sms)
    return m + (5 - m % TILE) % TILE


def boundary_lengths():
    """Row lengths at the kernels' lane-group edges: 1, G - 1, G, G + 1, 2G + 1 for every row kernel's G and every split
    kernel's GN (lanes across a row's entries), and the split kernels' GN * UN chunk lengths +- 1."""
    lens = {1}
    for g in set(ROW_G.values()) | {gn for _, gn, _ in SPLIT.values()}:
        lens |= {g - 1, g, g + 1, 2 * g + 1}
    for _, gn, un in SPLIT.values():
        lens |= {gn * un - 1, gn * un, gn * un + 1}
    lens.discard(0)
    return sorted(lens)


def row_lengths(M, min_nnz=0, seed=1):
    """The row-length profile: short random rows (many empty), with min_nnz entries at least; every boundary length
    at seven places spread over the rows; EMPTY_RUN empty rows from a tile boundary at three places; LONG_ROWS early,
    in the middle and late; the first and the last row non-empty."""
    rng = np.random.default_rng(seed)
    lens = rng.choice(np.array([0, 0, 0, 1, 2, 3, 4]), M)
    if min_nnz > lens.sum():
        lens += rng.integers(0, 2 * -(-(min_nnz - lens.sum()) // M) + 2, M)
    bl = np.array(boundary_lengths())
    for k, start in enumerate(np.linspace(16, M - len(bl) - 64, 7).astype(np.int64)):
        lens[start:start + len(bl)] = np.roll(bl, k)
    for frac in (0.2, 0.55, 0.9):
        start = int(M * frac) // TILE * TILE
        lens[start:start + EMPTY_RUN] = 0
    for at, n in zip((2, M // 2 + 3, M - 40, M - 3), LONG_ROWS):
        lens[at] = n
    lens[0], lens[M - 1] = 3, 2
    return lens


class Block:
    """A CSR block with the profile above: M rows, N != M columns, column N - 1 used, duplicate (row, col) pairs."""

    def __init__(self, M, min_nnz=0, seed=1):
        self.M, self.N = M, M // 2 + 77
        self.lens = row_lengths(M, min_nnz, seed)
        self.rowStart = np.zeros(M + 1, np.int64)
        np.cumsum(self.lens, out=self.rowStart[1:])
        self.nnz = int(self.rowStart[-1])
        rng = np.random.default_rng(seed + 1)
        self.col_idx = rng.integers(0, self.N, self.nnz)
        self.col_idx[::97] = self.N - 1
        self.col_idx[self.rowStart[0]:self.rowStart[1]] = [self.N - 1, 5, self.N - 1]
        two = np.flatnonzero(self.lens >= 2)[::5]  # a duplicate pair at the start of every fifth row of 2+ entries
        self.col_idx[self.rowStart[two] + 1] = self.col_idx[self.rowStart[two]]
        self.row_idx = np.repeat(np.arange(M, dtype=np.int64), self.lens)


def exact_bound(r, max_len):
    """The largest magnitude any partial sum of any case can reach (SpMM of scaled SDDMM results over the longest row);
    results are exact in fp64 while it stays below 2^53 / 4 (scales down to 1/4)."""
    dot = r * OPERAND.max() ** 2
    return max_len * (VMAX + dot) * SMAX * OPERAND.max() + VMAX


class Reference:
    """Integer operands of one block at width r and every expected output, exact; sparse products made on demand."""

    def __init__(self, blk, r, seed=7):
        import scipy.sparse as sp
        self.blk, self.r = blk, r
        rng = np.random.default_rng(seed * 1000 + r)
        self.X = rng.choice(OPERAND, (blk.M, r))
        self.Y = rng.choice(OPERAND, (blk.N, r))
        self.v0 = rng.integers(-VMAX, VMAX + 1, blk.nnz).astype(np.float64)
        self.w = rng.choice(OPERAND, blk.nnz)
        self.O0 = rng.integers(-VMAX, VMAX + 1, (blk.M, r)).astype(np.float64)
        self.scale = rng.choice(SCALES, blk.nnz)
        self.dots = np.empty(blk.nnz)
        step = max(1, (1 << 22) // r)
        for s in range(0, blk.nnz, step):
            e = min(s + step, blk.nnz)
            self.dots[s:e] = np.einsum("ij,ij->i", self.X[blk.row_idx[s:e]], self.Y[blk.col_idx[s:e]])
        self._sp = lambda vals: sp.csr_matrix((vals, blk.col_idx, blk.rowStart), shape=(blk.M, blk.N)) @ self.Y
        self._prod = {}

    def spmm(self, key):
        """S_vals @ Y for vals = w, dots, v0 + dots or scale * dots."""
        if key not in self._prod:
            vals = {"w": self.w, "dots": self.dots, "acc": self.v0 + self.dots, "scaled": self.scale * self.dots}[key]
            self._prod[key] = self._sp(vals)
        return self._prod[key]


def first_mismatch(name, got, want):
    """None when got is bit-equal to want (NaN nowhere), else a one-line description of the first difference."""
    got, want = np.asarray(got), np.asarray(want)
    if got.shape != want.shape:
        return f"{name}: shape {got.shape} != {want.shape}"
    bad = np.flatnonzero((got != want).ravel())
    if not len(bad):
        return None
    i = bad[0]
    where = np.unravel_index(i, got.shape)
    return f"{name}: {len(bad)} of {got.size} differ; first at {tuple(int(k) for k in where)}: got {got.ravel()[i]!r}, want {want.ravel()[i]!r}"


class Device:
    """The block and the operands of one width on the device; dense operands at an 8-byte offset when `offset`."""

    def __init__(self, ref, offset=False):
        import torch
        self.torch, self.ref, self.blk = torch, ref, ref.blk
        self.offset = 1 if offset else 0
        self.stream = torch.cuda.current_stream().cuda_stream
        self.rs = torch.from_numpy(self.blk.rowStart).cuda()
        self.ci = torch.from_numpy(self.blk.col_idx).cuda()
        self.X, self.pX = self.dense(ref.X)
        self.Y, self.pY = self.dense(ref.Y)

    def dense(self, a, fill=None):
        """(tensor, pointer): a copy of a, or an array of a's shape filled with `fill`, at the block's offset."""
        t = self.torch.full((a.size + self.offset,), np.nan if fill is None else fill, dtype=self.torch.float64, device="cuda")
        if fill is None:
            t[self.offset:] = self.torch.from_numpy(np.ascontiguousarray(a).ravel()).cuda()
        return t, t.data_ptr() + 8 * self.offset

    def host(self, t, shape):
        self.torch.cuda.synchronize()
        return t[self.offset:].cpu().numpy().reshape(shape)

    def vec(self, a=None, n=None):
        import torch
        if a is None:
            return torch.full((n,), float("nan"), dtype=torch.float64, device="cuda")
        return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _check(L, rc, what):
    if rc != 0:
        raise AssertionError(f"{what}: rc {rc}: {L.hnh_last_error_string().decode()}")


def check_group(L, sms, r, path, ops, flag_sets=(0,), offset=False, force=0, log=print):
    """Runs `ops` at width r on a block sized for `path`; returns the list of mismatches (empty: all bit-equal).
    flag_sets: the path-selecting flags each op runs under (TMA_STAGE, TMA_WARP, FORCE_DIRECT, ...); force: flags
    added to every call (FORCE_GENERIC)."""
    units = units_per_cta(path, r)
    M = rows_for(units, sms)
    assert M >= wave_bound(units, sms) and M % TILE != 0
    blk = _block(M)
    assert exact_bound(r, int(blk.lens.max())) < 2.0 ** 51
    ref = Reference(blk, r)
    dv = Device(ref, offset)
    errs = []
    nnz, M, N = blk.nnz, blk.M, blk.N

    def expect(name, got, want):
        e = first_mismatch(f"r={r} {path} {name}", got, want)
        if e:
            errs.append(e)
            log(e)

    for base in flag_sets:
        base |= force
        tag = f"flags={base}"
        if "sddmm" in ops:
            for fl, want in ((0, ref.v0 + ref.dots), (BETA0, ref.dots)):
                v = dv.vec(ref.v0) if fl == 0 else dv.vec(n=nnz)
                _check(L, L.hnh_sddmm_f64(dv.rs.data_ptr(), dv.ci.data_ptr(), v.data_ptr(), M, nnz, dv.pX, dv.pY, r, base | fl,
                                          dv.stream), "sddmm")
                expect(f"sddmm {tag}|{fl}", _host(dv, v), want)
        if "sddmm_scaled" in ops:
            acc, d0, sc = ref.v0 + ref.dots, ref.dots, ref.scale
            S = dv.vec(sc)
            cases = (("beta0 + scaled_out", BETA0, True, d0, sc * d0), ("beta0 + SCALE_VALUES", BETA0 | SCALE_VALUES, True, sc * d0, sc * d0),
                     ("beta0, no scaled_out", BETA0, False, sc * d0, None), ("accumulate + scaled_out", 0, True, acc, sc * acc))
            for name, fl, with_out, want_v, want_o in cases:
                v = dv.vec(ref.v0) if fl & BETA0 == 0 else dv.vec(n=nnz)
                o = dv.vec(n=nnz)
                _check(L, L.hnh_sddmm_scaled_f64(dv.rs.data_ptr(), dv.ci.data_ptr(), v.data_ptr(), M, nnz, dv.pX, dv.pY, r, base | fl,
                                                 S.data_ptr(), o.data_ptr() if with_out else None, dv.stream), "sddmm_scaled " + name)
                expect(f"sddmm_scaled {name} {tag} values", _host(dv, v), want_v)
                if with_out:
                    expect(f"sddmm_scaled {name} {tag} scaled_out", _host(dv, o), want_o)
            for fl, want_v in ((BETA0, d0), (BETA0 | SCALE_VALUES, sc * d0)):  # scaled_out == scale: the separate-pass fallback
                v, so = dv.vec(n=nnz), dv.vec(sc)
                _check(L, L.hnh_sddmm_scaled_f64(dv.rs.data_ptr(), dv.ci.data_ptr(), v.data_ptr(), M, nnz, dv.pX, dv.pY, r, base | fl,
                                                 so.data_ptr(), so.data_ptr(), dv.stream), "sddmm_scaled aliased")
                expect(f"sddmm_scaled scaled_out == scale {tag}|{fl} values", _host(dv, v), want_v)
                expect(f"sddmm_scaled scaled_out == scale {tag}|{fl} scaled_out", _host(dv, so), sc * d0)
        if "spmm" in ops:
            w = dv.vec(ref.w)
            for fl, want in ((0, ref.O0 + ref.spmm("w")), (BETA0, ref.spmm("w"))):
                out, p = dv.dense(ref.O0) if fl == 0 else dv.dense(ref.O0, np.nan)
                _check(L, L.hnh_spmm_f64(dv.rs.data_ptr(), dv.ci.data_ptr(), w.data_ptr(), M, nnz, dv.pY, p, r, base | fl, dv.stream),
                       "spmm")
                expect(f"spmm {tag}|{fl}", dv.host(out, (M, r)), want)
        if "fused" in ops:
            for fl in (0, BETA0, BETA0_VALUES, BETA0_OUT):
                bv, bo = bool(fl & (BETA0 | BETA0_VALUES)), bool(fl & (BETA0 | BETA0_OUT))
                v = dv.vec(n=nnz) if bv else dv.vec(ref.v0)
                out, p = dv.dense(ref.O0, np.nan) if bo else dv.dense(ref.O0)
                _check(L, L.hnh_fused_f64(dv.rs.data_ptr(), dv.ci.data_ptr(), v.data_ptr(), M, nnz, dv.pX, dv.pY, p, r, base | fl,
                                          dv.stream), "fused")
                expect(f"fused {tag}|{fl} values", _host(dv, v), ref.dots if bv else ref.v0 + ref.dots)
                prod = ref.spmm("dots" if bv else "acc")
                expect(f"fused {tag}|{fl} Out", dv.host(out, (M, r)), prod if bo else ref.O0 + prod)
        if "fused_inplace" in ops:  # Out == X
            for fl in (BETA0, BETA0_OUT):
                bv = fl == BETA0
                v = dv.vec(n=nnz) if bv else dv.vec(ref.v0)
                xo, p = dv.dense(ref.X)
                _check(L, L.hnh_fused_f64(dv.rs.data_ptr(), dv.ci.data_ptr(), v.data_ptr(), M, nnz, p, dv.pY, p, r, base | fl,
                                          dv.stream), "fused in place")
                expect(f"fused in place {tag}|{fl} values", _host(dv, v), ref.dots if bv else ref.v0 + ref.dots)
                expect(f"fused in place {tag}|{fl} Out", dv.host(xo, (M, r)), ref.spmm("dots" if bv else "acc"))
        if "fused_scaled" in ops:
            S = dv.vec(ref.scale)
            want_v = ref.scale * ref.dots
            for fl in (BETA0_VALUES, BETA0_VALUES | BETA0_OUT):
                bo = bool(fl & BETA0_OUT)
                v, so = dv.vec(n=nnz), dv.vec(n=nnz)
                out, p = dv.dense(ref.O0, np.nan) if bo else dv.dense(ref.O0)
                _check(L, L.hnh_fused_scaled_f64(dv.rs.data_ptr(), dv.ci.data_ptr(), v.data_ptr(), M, nnz, dv.pX, dv.pY, p, r,
                                                 base | fl, S.data_ptr(), so.data_ptr(), dv.stream), "fused_scaled")
                expect(f"fused_scaled {tag}|{fl} values", _host(dv, v), want_v)
                expect(f"fused_scaled {tag}|{fl} scaled_out", _host(dv, so), want_v)
                expect(f"fused_scaled {tag}|{fl} Out", dv.host(out, (M, r)), ref.spmm("scaled") if bo else ref.O0 + ref.spmm("scaled"))
    return errs


def check_coo(L, sms, r, force=0, log=print):
    """hnh_sddmm_coo_f64 with at least WAVES iterations of COO_UNIT entries per CTA."""
    need = wave_bound(COO_UNIT, sms)
    blk = _block(rows_for(TILE, sms), min_nnz=need)
    assert blk.nnz >= need
    ref = Reference(blk, r)
    dv = Device(ref)
    ri = dv.torch.from_numpy(blk.row_idx).cuda()
    v = dv.vec(ref.v0)
    _check(L, L.hnh_sddmm_coo_f64(ri.data_ptr(), dv.ci.data_ptr(), v.data_ptr(), blk.nnz, dv.pX, dv.pY, r, force, dv.stream),
           "sddmm_coo")
    e = first_mismatch(f"r={r} coo flags={force}", _host(dv, v), ref.v0 + ref.dots)
    if e:
        log(e)
    return [e] if e else []


def _host(dv, t):
    dv.torch.cuda.synchronize()
    return t.cpu().numpy()


_BLOCKS = {}


def _block(M, min_nnz=0):
    if (M, min_nnz) not in _BLOCKS:
        _BLOCKS.clear()  # one block alive at a time
        _BLOCKS[(M, min_nnz)] = Block(M, min_nnz)
    return _BLOCKS[(M, min_nnz)]


ALL_OPS = ("sddmm", "sddmm_scaled", "spmm", "fused", "fused_inplace", "fused_scaled")
# groups run in a child process: (environment, [(r, path, ops, flag_sets)])
ENV_GROUPS = {
    # the direct-load row kernels at the split widths
    "split_max_r_0": ({"HNH_SPLIT_MAX_R": "0"}, [(r, "row", ALL_OPS, (0,)) for r in (4, 8, 16, 32)]),
    # split kernels up to 16, the row kernel at 32
    "split_max_r_16": ({"HNH_SPLIT_MAX_R": "16"}, [(16, "split", ALL_OPS, (0,)), (32, "row", ALL_OPS, (0,))]),
    # TMA staging everywhere it applies: the fused kernel at r = 128 and the accumulating fused kernel at 256 as well
    "tma_1": ({"HNH_TMA": "1"}, [(r, "tma", ("sddmm", "sddmm_scaled", "fused"), (0,)) for r in (128, 256)]),
    # direct loads everywhere: SDDMM at r = 128 and 256 and the overwriting fused kernel at 256
    "tma_0": ({"HNH_TMA": "0"}, [(r, "row", ("sddmm", "sddmm_scaled", "fused"), (0,)) for r in (128, 256)]),
}


def run_env_group(name):
    """Child-process entry: the group's environment must already be set.  Returns the process exit code."""
    import torch
    from distributed_sddmm_b200 import lib
    env, groups = ENV_GROUPS[name]
    for k, v in env.items():
        assert os.environ.get(k) == v, f"{name}: run with {k}={v}"
    L = lib()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    errs = []
    for r, path, ops, flag_sets in groups:
        errs += check_group(L, sms, r, path, ops, flag_sets)
        if errs:
            break
    print(f"{name}: {'FAILED' if errs else 'ok'} ({len(groups)} widths, {sms} SMs)")
    return 1 if errs else 0


if __name__ == "__main__":
    sys.exit(run_env_group(sys.argv[1]))
