"""The fused SDDMM -> SpMM kernel at the G = 32 widths (r = 64, 128, 256), whose direct form stages the gathered rows
through a per-warp ring of cp.async slots that runs across row ends: bit-exact against numpy / scipy on the exact-
integer operands of tests/kernel_waves_worker.py, and bit-equal to the TMA-staged fused kernels where those exist.

The row lengths are drawn from the lengths where a batch, the ring, a chunk of 32 column indices or a row ends (0, 1,
batch -1 / +0 / +1, 32, 33, 64 and longer), with runs of empty rows between long rows, over more rows than one resident
wave of warps holds, so that every warp's ring crosses many row ends and refills across empty rows."""
import numpy as np
import pytest
import torch

from tests import kernel_waves_worker as kw

pytestmark = pytest.mark.gpu

WIDTHS = [64, 128, 256]
# lengths at the batch (1 or 2 rows), ring (up to 12 rows) and 32-entry chunk edges, and long rows
LENGTHS = np.array([0, 1, 2, 3, 4, 5, 6, 7, 8, 11, 12, 13, 31, 32, 33, 64, 65, 97, 130])


class RingBlock:
    """kw.Block's attributes with the ring's row-length profile: M rows, N != M columns, column N - 1 used."""

    def __init__(self, M, seed=3):
        rng = np.random.default_rng(seed)
        self.M, self.N = M, M // 2 + 77
        lens = rng.choice(LENGTHS, M)
        lens[rng.random(M) < 0.3] = 0  # many empty rows
        for start in range(64, M - 16, M // 9):  # long, empty x 5, long, empty x 5, ...
            lens[start:start + 12] = [200, 0, 0, 0, 0, 0, 150, 0, 0, 0, 0, 0]
        lens[0], lens[M - 1] = 33, 1
        self.lens = lens
        self.rowStart = np.zeros(M + 1, np.int64)
        np.cumsum(lens, out=self.rowStart[1:])
        self.nnz = int(self.rowStart[-1])
        self.col_idx = np.random.default_rng(seed + 1).integers(0, self.N, self.nnz)
        self.col_idx[::89] = self.N - 1
        self.row_idx = np.repeat(np.arange(M, dtype=np.int64), lens)


@pytest.fixture(scope="module")
def block():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    # two of the largest grid's full waves of one-warp rows: every warp takes at least 2 * WAVES rows
    blk = RingBlock(2 * kw.rows_for(kw.units_per_cta("row", 128), sms))
    assert kw.exact_bound(256, int(blk.lens.max())) < 2.0 ** 51
    return blk


def _check(L, rc, what):
    assert rc == 0, f"{what}: rc {rc}: {L.hnh_last_error_string().decode()}"


def _fused(L, dv, r, flags, v, p_x, p_out):
    blk = dv.blk
    _check(L, L.hnh_fused_f64(dv.rs.data_ptr(), dv.ci.data_ptr(), v.data_ptr(), blk.M, blk.nnz, p_x, dv.pY, p_out, r,
                              flags, dv.stream), f"fused r={r} flags={flags}")


@pytest.mark.parametrize("r", WIDTHS)
def test_fused_ring_every_form_matches_oracle(hnh, block, r):
    """The four overwrite forms (values and Out accumulated or overwritten), out of place, on the direct kernel."""
    ref = kw.Reference(block, r)
    dv = kw.Device(ref)
    M, nnz = block.M, block.nnz
    errs = []
    for fl in (0, kw.BETA0, kw.BETA0_VALUES, kw.BETA0_OUT):
        bv, bo = bool(fl & (kw.BETA0 | kw.BETA0_VALUES)), bool(fl & (kw.BETA0 | kw.BETA0_OUT))
        v = dv.vec(n=nnz) if bv else dv.vec(ref.v0)
        out, p = dv.dense(ref.O0, np.nan) if bo else dv.dense(ref.O0)
        _fused(hnh, dv, r, kw.FORCE_DIRECT | fl, v, dv.pX, p)
        prod = ref.spmm("dots" if bv else "acc")
        for e in (kw.first_mismatch(f"r={r} flags={fl} values", kw._host(dv, v), ref.dots if bv else ref.v0 + ref.dots),
                  kw.first_mismatch(f"r={r} flags={fl} Out", dv.host(out, (M, r)), prod if bo else ref.O0 + prod)):
            if e:
                errs.append(e)
    torch.cuda.empty_cache()
    assert not errs, "\n".join(errs)


@pytest.mark.parametrize("r", WIDTHS)
def test_fused_ring_in_place_and_scaled_match_oracle(hnh, block, r):
    """Out == X (the one-GPU FusedMM's form), and the scaled epilogue with Out accumulated and overwritten."""
    ref = kw.Reference(block, r)
    dv = kw.Device(ref)
    M, nnz = block.M, block.nnz
    errs = []
    for fl in (kw.BETA0, kw.BETA0_OUT):
        bv = fl == kw.BETA0
        v = dv.vec(n=nnz) if bv else dv.vec(ref.v0)
        xo, p = dv.dense(ref.X)
        _fused(hnh, dv, r, fl, v, p, p)
        errs += [kw.first_mismatch(f"r={r} in place flags={fl} values", kw._host(dv, v), ref.dots if bv else ref.v0 + ref.dots),
                 kw.first_mismatch(f"r={r} in place flags={fl} Out", dv.host(xo, (M, r)), ref.spmm("dots" if bv else "acc"))]
    S = dv.vec(ref.scale)
    want_v = ref.scale * ref.dots
    for fl in (kw.BETA0_VALUES, kw.BETA0_VALUES | kw.BETA0_OUT):
        bo = bool(fl & kw.BETA0_OUT)
        v, so = dv.vec(n=nnz), dv.vec(n=nnz)
        out, p = dv.dense(ref.O0, np.nan) if bo else dv.dense(ref.O0)
        _check(hnh, hnh.hnh_fused_scaled_f64(dv.rs.data_ptr(), dv.ci.data_ptr(), v.data_ptr(), M, nnz, dv.pX, dv.pY, p, r, fl,
                                             S.data_ptr(), so.data_ptr(), dv.stream), f"fused_scaled r={r} flags={fl}")
        errs += [kw.first_mismatch(f"r={r} scaled flags={fl} values", kw._host(dv, v), want_v),
                 kw.first_mismatch(f"r={r} scaled flags={fl} scaled_out", kw._host(dv, so), want_v),
                 kw.first_mismatch(f"r={r} scaled flags={fl} Out", dv.host(out, (M, r)),
                                   ref.spmm("scaled") if bo else ref.O0 + ref.spmm("scaled"))]
    torch.cuda.empty_cache()
    errs = [e for e in errs if e]
    assert not errs, "\n".join(errs)


@pytest.mark.parametrize("r", [128, 256])
def test_fused_ring_bit_equal_to_tma_kernels(hnh, block, r):
    """Direct (ring) and TMA-staged fused kernels, same inputs, every overwrite form: identical bits."""
    ref = kw.Reference(block, r)
    dv = kw.Device(ref)
    M, nnz = block.M, block.nnz
    for fl in (0, kw.BETA0, kw.BETA0_VALUES, kw.BETA0_OUT):
        bv, bo = bool(fl & (kw.BETA0 | kw.BETA0_VALUES)), bool(fl & (kw.BETA0 | kw.BETA0_OUT))
        got = []
        for path in (kw.FORCE_DIRECT, kw.TMA_STAGE):
            v = dv.vec(n=nnz) if bv else dv.vec(ref.v0)
            out, p = dv.dense(ref.O0, np.nan) if bo else dv.dense(ref.O0)
            _fused(hnh, dv, r, path | fl, v, dv.pX, p)
            got.append((kw._host(dv, v), dv.host(out, (M, r))))
        (v_ring, o_ring), (v_tma, o_tma) = got
        assert np.array_equal(v_ring, v_tma) and np.array_equal(o_ring, o_tma), f"r={r} flags={fl}"
    torch.cuda.empty_cache()
