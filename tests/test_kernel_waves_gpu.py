"""The SDDMM / SpMM / fused engine past one resident wave, bit-exact against numpy / scipy on the row-length profile
of tests/kernel_waves_worker.py: every path the dispatch offers (split, direct-load row, TMA-staged, per-warp TMA,
generic, unaligned operands, COO) under every overwrite flag, in place and with the scale epilogues.  Each case is
sized from the device's SM count so that every CTA runs at least three grid-stride iterations.

The paths that HNH_SPLIT_MAX_R and HNH_TMA select run in a child process each: the library reads both once per
process."""
import os
import subprocess
import sys

import pytest
import torch

from tests import kernel_waves_worker as kw

pytestmark = pytest.mark.gpu

ALL = kw.ALL_OPS


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _run(hnh, sms, r, path, ops, flag_sets=(0,), **kw_):
    errs = kw.check_group(hnh, sms, r, path, ops, flag_sets, **kw_)
    torch.cuda.empty_cache()
    assert not errs, "\n".join(errs[:10])


@pytest.mark.parametrize("r", [4, 8, 16, 32])
def test_split_kernels_past_one_wave(hnh, sms, r):
    _run(hnh, sms, r, "split", ALL)


def test_row_kernel_r64_past_one_wave(hnh, sms):
    _run(hnh, sms, 64, "row", ALL)


@pytest.mark.parametrize("r", [128, 256])
def test_r128_r256_every_path_past_one_wave(hnh, sms, r):
    """Default dispatch (TMA-staged SDDMM, direct fused at 128, TMA fused at 256 when Out is overwritten), then each
    path forced: direct loads, TMA staging, per-warp TMA.  All take one 8-row tile per CTA iteration."""
    _run(hnh, sms, r, "tma", ("sddmm", "sddmm_scaled", "fused"), (0, kw.TMA_STAGE, kw.TMA_WARP, kw.FORCE_DIRECT))
    _run(hnh, sms, r, "row", ("spmm", "fused_inplace", "fused_scaled"))


@pytest.mark.parametrize("r,force,offset", [(12, 0, False), (100, 0, False), (64, kw.FORCE_GENERIC, False), (32, 0, True)],
                         ids=["r12", "r100", "forced", "unaligned"])
def test_generic_kernels_past_one_wave(hnh, sms, r, force, offset):
    """The any-r one-warp-per-row kernels: widths outside the table, FORCE_GENERIC, and operands 8-byte aligned only;
    the scaled SDDMM takes its separate-pass fallback there."""
    _run(hnh, sms, r, "generic", ("sddmm", "sddmm_scaled", "spmm", "fused"), force=force, offset=offset)


@pytest.mark.parametrize("r,force", [(r, 0) for r in kw.TABLE] + [(12, 0), (128, kw.FORCE_GENERIC)])
def test_sddmm_coo_past_one_wave(hnh, sms, r, force):
    errs = kw.check_coo(hnh, sms, r, force)
    torch.cuda.empty_cache()
    assert not errs, errs


@pytest.mark.parametrize("group", sorted(kw.ENV_GROUPS))
def test_environment_selected_paths_past_one_wave(group):
    """HNH_SPLIT_MAX_R = 0 (row kernels at r = 4..32) and 16, HNH_TMA = 1 and 0, each in its own process."""
    env = dict(os.environ, **kw.ENV_GROUPS[group][0])
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-m", "tests.kernel_waves_worker", group]
    p = subprocess.run(cmd, cwd=kw.ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-4000:]
    assert f"{group}: ok" in p.stdout
