"""tests/test_zz_r_shard_scan_gpu.py - dann_shards_scan: the per-shard rescans, the many-index first round, the
host-side merge and its worker threads - run on the CPU against the product's C ABI built for the SIMT emulator (see
tests/test_emulated_abi.py) with two fake devices, under the default lane order and in shuffled fiber order."""
import pytest

from test_emulated_abi import _run

N_TESTS = 39     # every test of tests/test_zz_r_shard_scan_gpu.py, parameter sets included


@pytest.mark.parametrize("sched", [None, "2"], ids=["default_order", "shuffled"])
def test_shard_scan_suite_passes_under_emulation(sched):
    env = {"SIMT_FAKE_DEVICES": "2"}
    if sched:
        env["SIMT_SCHED"] = sched
    passed, out = _run(["tests/test_zz_r_shard_scan_gpu.py"], env)
    assert passed == N_TESTS and "skipped" not in out.splitlines()[-1], out[-500:]
