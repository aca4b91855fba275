"""tests/test_zz_u_scan_fetch_gpu.py - dann_scan_fetch against single amgettuple calls and the oracle: every fetch size,
layout, regrow, deep growth, interleaving and special value there - run on the CPU against the product's C ABI built for
the SIMT emulator (see tests/test_emulated_abi.py), under the default lane order and in shuffled fiber order."""
import pytest

from test_emulated_abi import _run

N_TESTS = 23     # every test of tests/test_zz_u_scan_fetch_gpu.py, parameter sets included


@pytest.mark.parametrize("sched", [None, "2"], ids=["default_order", "shuffled"])
def test_scan_fetch_suite_passes_under_emulation(sched):
    passed, out = _run(["tests/test_zz_u_scan_fetch_gpu.py"], {"SIMT_SCHED": sched} if sched else None)
    assert passed == N_TESTS and "skipped" not in out.splitlines()[-1], out[-500:]
