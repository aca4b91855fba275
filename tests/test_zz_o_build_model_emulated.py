"""tests/test_zz_o_build_model_gpu.py - dann_build_graph edge for edge against the CPU model of the batched build - run
on the CPU against the product's C ABI built for the SIMT emulator (see tests/test_emulated_abi.py), under the default
lane order and in shuffled fiber order.  The 40 000-node case is left to hardware."""
import pytest

from test_emulated_abi import _run

N_TESTS = 41     # every test of tests/test_zz_o_build_model_gpu.py but the hardware-only one, parameter sets included


@pytest.mark.parametrize("sched", [None, "2"], ids=["default_order", "shuffled"])
def test_build_model_suite_passes_under_emulation(sched):
    passed, out = _run(["tests/test_zz_o_build_model_gpu.py", "-k", "not hardware_only"], {"SIMT_SCHED": sched} if sched else None)
    assert passed == N_TESTS and "skipped" not in out.splitlines()[-1], out[-500:]
