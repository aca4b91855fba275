"""tests/test_zz_s_deep_scan_gpu.py - the streaming scan's deep mode: its entry from every planned layout, in-place
growth, rescans, the many-scan rounds, the coalescer and the sharded scan - run on the CPU against the product's C ABI
built for the SIMT emulator (see tests/test_emulated_abi.py), under the default lane order and in shuffled fiber
order.  The 300 000-node drain without hooks is hardware only: it is the one test skipped here."""
import pytest

from test_emulated_abi import _run

N_TESTS = 13     # every test of tests/test_zz_s_deep_scan_gpu.py but the hardware drain, parameter sets included


@pytest.mark.parametrize("sched", [None, "2"], ids=["default_order", "shuffled"])
def test_deep_scan_suite_passes_under_emulation(sched):
    passed, out = _run(["tests/test_zz_s_deep_scan_gpu.py"], {"SIMT_SCHED": sched} if sched else None)
    assert passed == N_TESTS and "1 skipped" in out.splitlines()[-1], out[-500:]
