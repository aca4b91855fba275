"""tests/test_zz_q_shards_gpu.py - dann_shards: every shard's batch, the worker threads, the peer copies and the merge
kernel - run on the CPU against the product's C ABI built for the SIMT emulator (see tests/test_emulated_abi.py) with
two fake devices, under the default lane order and in shuffled fiber order."""
import pytest

from test_emulated_abi import _run

N_TESTS = 35     # every test of tests/test_zz_q_shards_gpu.py, parameter sets included


@pytest.mark.parametrize("sched", [None, "2"], ids=["default_order", "shuffled"])
def test_shards_suite_passes_under_emulation(sched):
    env = {"SIMT_FAKE_DEVICES": "2"}
    if sched:
        env["SIMT_SCHED"] = sched
    passed, out = _run(["tests/test_zz_q_shards_gpu.py"], env)
    assert passed == N_TESTS and "skipped" not in out.splitlines()[-1], out[-500:]
