"""tests/test_zz_n_scan_many_gpu.py - dann_scan_gettuple_many, its kernels and the coalescer's gettuple dispatch - run
on the CPU against the product's C ABI built for the SIMT emulator (see tests/test_emulated_abi.py), under the default
lane order and in shuffled fiber order."""
import pytest

from test_emulated_abi import _run

N_TESTS = 19     # every test of tests/test_zz_n_scan_many_gpu.py, parameter sets included


@pytest.mark.parametrize("sched", [None, "2"], ids=["default_order", "shuffled"])
def test_scan_many_suite_passes_under_emulation(sched):
    passed, out = _run(["tests/test_zz_n_scan_many_gpu.py"], {"SIMT_SCHED": sched} if sched else None)
    assert passed == N_TESTS and "skipped" not in out.splitlines()[-1], out[-500:]
