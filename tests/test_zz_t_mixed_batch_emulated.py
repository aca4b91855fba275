"""tests/test_zz_t_mixed_batch_gpu.py - dann_search_batch_mixed, its device and group entry points and the coalescer's
mixed dispatch - run on the CPU against the product's C ABI built for the SIMT emulator (see tests/test_emulated_abi.py),
under the default lane order and in shuffled fiber order, with two fake devices so that the group case runs too."""
import pytest

from test_emulated_abi import _run

N_TESTS = 19     # every test of tests/test_zz_t_mixed_batch_gpu.py, parameter sets included


@pytest.mark.parametrize("sched", [None, "2"], ids=["default_order", "shuffled"])
def test_mixed_batch_suite_passes_under_emulation(sched):
    env = {"SIMT_FAKE_DEVICES": "2"}
    if sched:
        env["SIMT_SCHED"] = sched
    passed, out = _run(["tests/test_zz_t_mixed_batch_gpu.py"], env)
    assert passed == N_TESTS and "skipped" not in out.splitlines()[-1], out[-500:]
