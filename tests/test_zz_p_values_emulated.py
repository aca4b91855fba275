"""tests/test_zz_p_values_gpu.py - the scan path on extreme, degenerate and multi-bit values - run on the CPU against
the product's C ABI built for the SIMT emulator (see tests/test_emulated_abi.py), under the default lane order and in
shuffled fiber order.

The emulator runs x86 float arithmetic, so this run cannot see what only the GPU's float unit does: the bits of a NaN
inner product (x86 gives the reference's 0x7FC00000 whether or not full_distance_group8 maps it) and whether subnormals
are flushed to zero (a build with -ftz=true).  It does pin the quantizer's branches, the multi-bit packing and the
tie order on these values."""
import pytest

from test_emulated_abi import _run

N_TESTS = 21     # every test of tests/test_zz_p_values_gpu.py, parameter sets included


@pytest.mark.parametrize("sched", [None, "2"], ids=["default_order", "shuffled"])
def test_values_suite_passes_under_emulation(sched):
    passed, out = _run(["tests/test_zz_p_values_gpu.py"], {"SIMT_SCHED": sched} if sched else None)
    assert passed == N_TESTS and "skipped" not in out.splitlines()[-1], out[-500:]
