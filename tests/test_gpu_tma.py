"""GPU parity of the TMA pipeline variant of the tick kernel (`SERFSIM_TMA=1`: cp.async.bulk + mbarrier staging of whole
tiles, single-slot unsharded runs).  It is device-only code — tests/emu compiles it out — so these device runs are the
only evidence for it: the same comparisons as tests/test_gpu_parity.py (records, clocks, every trace row, hashes,
trace on and off) against the CPU oracle, with the variant switched on and a check that it really was selected."""
import os

import pytest

import parity_lib as P
from serf_b200 import GossipSim, scenarios

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _tma(monkeypatch):
    monkeypatch.setenv("SERFSIM_TMA", "1")
    monkeypatch.setenv("SERFSIM_VERBOSE", "1")


def _selected(capfd):
    err = capfd.readouterr().err
    if os.environ.get("SERFSIM_GPU_TESTS_ON_EMU"):        # dry run of the test code on the host build: the TMA kernel is compiled out there
        return True
    return "tick kernel = tick_kernel_tma" in err


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_tma_config1_random_graph_100k(seed, capfd):
    P.run_against_oracle(GossipSim, scenarios.random_graph_leave(100_000, 16, 3, seed))
    assert _selected(capfd)


def test_tma_fanout4_ragged_tail(capfd):
    P.run_against_oracle(GossipSim, scenarios.random_graph_leave(60_001, 12, 4, seed=5))          # last tile partly filled
    assert _selected(capfd)


def test_tma_failure_detection(capfd):
    sc = scenarios.random_graph_fail(20_000, 16, 3, seed=2)
    sc.slots, sc.subjects, sc.ops = 1, sc.subjects[:1], [op for op in sc.ops if op[2] == int(sc.subjects[0])]
    P.run_against_oracle(GossipSim, sc, suspicion_mult=2, suspicion_max_timeout_mult=2, probe_interval_ticks=2)
    assert _selected(capfd)


@pytest.mark.parametrize("seed", range(12))
def test_tma_fuzz_single_slot(seed, capfd):
    sc = scenarios.fuzz(seed, slots=1)
    sc.max_ticks = 1500
    P.run_against_oracle(GossipSim, sc)
    assert _selected(capfd)
