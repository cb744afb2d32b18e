"""The fixtures of the past-one-wave GPU tests, checked without a GPU: the row-length profile holds every boundary
it claims, the operands keep every result exact in fp64, and the wave arithmetic uses the launchers' own constants
(read back from csrc/launch.h, csrc/row_gather.cuh, csrc/c_abi.cu, csrc/edge_softmax.cu and csrc/gat_additive.cu)."""
import os
import re

import numpy as np
import pytest

from tests import test_attention_waves_gpu as aw
from tests import kernel_waves_worker as kw

CSRC = os.path.join(kw.ROOT, "distributed_sddmm_b200", "csrc")
SMS = 132  # H100 SXM; the arithmetic is checked for other SM counts too


def _src(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _macro(src, name):
    m = re.search(r"#define %s\(r, CALL(?:, FALLBACK)?\)(.*?)default:" % name, src, re.S)
    assert m, name
    return {int(a[0]): tuple(int(x) for x in a[1:]) for a in re.findall(r"case (\d+):\s*CALL\((\d+), (\d+), (\d+), (\d+)(?:, (\d+))?\)", m.group(1))
            for a in [tuple(x for x in a if x != "")]}


def test_dispatch_tables_match_the_shared_launch_path():
    launch, src = _src("launch.h"), _src("c_abi.cu")
    assert re.search(r"constexpr int kBlock = (\d+);", launch).group(1) == str(kw.BLOCK)
    split = _macro(src, "HNH_DISPATCH_SPLIT")
    assert {r: (gk, gn, un) for r, (_, gk, gn, _, un) in split.items()} == kw.SPLIT
    row = _macro(_src("row_gather.cuh"), "HNH_DISPATCH_R")
    assert {r: g for r, (_, g, _, _) in row.items()} == kw.ROW_G
    # work per CTA iteration: kBlock / G rows (row kernels), kBlock / (GK * GN) (split), 8-row tiles (TMA), one row per
    # warp (generic), kBlock / G groups of G entries (COO)
    assert src.count("per_cta = kBlock / G;") == 3 and src.count("grid_for(k, rows, per_cta, &grid);") == 3
    assert src.count("per_cta = kBlock / (GK * GN);") == 3
    assert src.count("grid_for(k, rows, %d, &grid)" % kw.TILE) == 2
    assert "grid_for(sddmm_generic_kernel, rows, kBlock / 32, &grid)" in src
    assert "grid_for(k, nnz, (int64_t)(kBlock / G) * G, &grid)" in src
    assert "constexpr int G = 32, VW = 2, TR = %d;" % kw.TILE in _src("kernels.cuh")
    # grid_for never launches more than SMs x occupancy CTAs unless given a smaller per-SM count (the calls above are
    # not), and a 2048-thread SM holds at most 8 CTAs of 256
    assert "int per_sm = kResident" in launch
    assert "cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kBlock, 0)" in launch
    assert "(int64_t)sms * per_sm" in launch
    assert "kCtasPerSm" not in src
    assert kw.CTAS_PER_SM * kw.BLOCK == 2048


def test_attention_grid_caps_match_the_shared_launch_path():
    assert "constexpr int kBlock = %d;" % aw.THREADS in _src("launch.h")
    for name in ("edge_softmax.cu", "gat_additive.cu"):
        src = _src(name)
        assert "constexpr int kCtasPerSm = %d;" % aw.GRID_PER_SM in src, name
        # every grid of the file is capped at kCtasPerSm per SM, and every launch has kBlock threads
        assert src.count("grid_for(") == src.count("&grid, kCtasPerSm)") > 0, name
        assert src.count("launch(") == src.count(", grid, kBlock, ") > 0, name
    assert "constexpr int kPiece = %d;" % aw.PIECE in _src("edge_softmax.cu")


@pytest.mark.parametrize("sms", [SMS, 114, 7])
def test_wave_arithmetic(sms):
    for path, r, units in (("split", 4, 16), ("split", 32, 8), ("row", 4, 128), ("row", 32, 16), ("row", 256, 8), ("tma", 128, 8),
                           ("generic", 12, 8), ("coo", 64, 256)):
        assert kw.units_per_cta(path, r) == units, (path, r)
        M = kw.rows_for(units, sms)
        grid = min(-(-M // units), sms * kw.CTAS_PER_SM)  # grid_for's largest possible grid
        assert M // (grid * units) >= kw.WAVES and M % kw.TILE == 5, (path, r)
    # the edge softmax and additive-attention kernels: warps per piece / row, threads per entry
    b = aw.bounds(sms)
    assert b["warps"] == aw.WAVES * aw.GRID_PER_SM * sms * aw.THREADS // 32
    assert b["threads"] == aw.WAVES * aw.GRID_PER_SM * sms * aw.THREADS


def test_row_length_profile():
    for M, min_nnz in ((kw.rows_for(8, SMS), 0), (kw.rows_for(128, SMS), 0), (kw.rows_for(8, SMS), kw.wave_bound(kw.COO_UNIT, SMS))):
        blk = kw.Block(M, min_nnz)
        lens = blk.lens
        assert blk.nnz >= min_nnz and blk.rowStart[-1] == blk.nnz and np.all(np.diff(blk.rowStart) == lens)
        assert M % kw.TILE != 0 and blk.N != M
        assert lens[0] > 0 and lens[-1] > 0
        have = set(lens.tolist())
        want = {1}
        for g in set(kw.ROW_G.values()) | {gn for _, gn, _ in kw.SPLIT.values()}:
            want |= {g - 1, g, g + 1, 2 * g + 1}
        for _, gn, un in kw.SPLIT.values():
            want |= {gn * un - 1, gn * un, gn * un + 1}
        want.discard(0)
        assert want <= have and want == set(kw.boundary_lengths())
        # each boundary length in the first and the last fifth of the rows: different grid-stride iterations
        for part in (lens[:M // 5], lens[-(M // 5):]):
            assert want <= set(part.tolist())
        # runs of >= 8 empty rows covering whole 8-row tiles
        empty_tiles = np.flatnonzero(lens[:M // kw.TILE * kw.TILE].reshape(-1, kw.TILE).sum(1) == 0)
        assert len(empty_tiles) >= 6
        # long rows early and late
        long_at = np.flatnonzero(lens >= 1000)
        assert len(long_at) >= 3 and long_at[0] < 16 and long_at[-1] > M - 64 and lens.max() <= 20000
        # duplicate (row, col) pairs and the last column
        key = blk.row_idx * blk.N + blk.col_idx
        assert len(np.unique(key)) < blk.nnz
        assert blk.col_idx.max() == blk.N - 1 and blk.col_idx.min() >= 0


def test_exactness_bound():
    """Every partial sum of every case stays below 2^51: integer-valued and quarter-valued results stay exact."""
    blk = kw.Block(kw.rows_for(8, SMS))
    for r in kw.TABLE + [12, 100]:
        assert kw.exact_bound(r, int(blk.lens.max())) < 2.0 ** 51
    ref = kw.Reference(kw.Block(1001), 32)
    for a in (ref.X, ref.Y, ref.w):
        assert np.all(a == np.rint(a)) and np.all(a != 0) and np.abs(a).max() <= kw.OPERAND.max()
    assert np.all(ref.v0 == np.rint(ref.v0)) and np.abs(ref.v0).max() <= kw.VMAX
    assert np.all(np.log2(np.abs(ref.scale)) == np.rint(np.log2(np.abs(ref.scale)))) and np.abs(ref.scale).max() <= kw.SMAX
    # the chunked reference dot products equal a plain loop
    want = np.array([ref.X[i] @ ref.Y[j] for i, j in zip(ref.blk.row_idx, ref.blk.col_idx)])
    assert np.array_equal(ref.dots, want)
    assert np.array_equal(ref.spmm("w"), ref.spmm("w"))
    dense = np.zeros((ref.blk.M, ref.blk.N))
    np.add.at(dense, (ref.blk.row_idx, ref.blk.col_idx), ref.w)
    assert np.array_equal(ref.spmm("w"), dense @ ref.Y)


def test_first_mismatch_reports():
    a = np.zeros((3, 2))
    assert kw.first_mismatch("x", a, a.copy()) is None
    b = a.copy()
    b[1, 1] = np.nan
    assert "(1, 1)" in kw.first_mismatch("x", b, a)
    assert "shape" in kw.first_mismatch("x", a, a[:2])


def test_attention_profile():
    for sms in (SMS, 7):
        keys, M = aw.softmax_keys(sms)
        b = aw.bounds(sms)
        lens = np.bincount(keys, minlength=M)
        pieces = int(np.sum(-(-lens // aw.PIECE)))
        assert M >= b["warps"] and pieces >= b["warps"] and len(keys) >= b["threads"]
        assert {1023, 1024, 1025, 2048, 2049} <= set(lens.tolist()) and (lens == 0).any()
