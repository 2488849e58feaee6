"""Unsharded sends read the destination words first and skip every RED.MAX that cannot raise its word (SERFSIM_DEDUP, on by
default).  On the host build of the kernels, with the filter on and off: records, clocks, trace rows and their hash, and stats
equal the oracle's, and SFS_PROBE 22 (skipped REDs) shows that the filter ran, or did not."""
import ctypes as C

import pytest

import envelope_lib as E
import parity_lib as P
from emu_lib import emu_sim, lib
from serf_b200.sim import random_regular_graph


@pytest.mark.parametrize("dedup", ["1", "0"])
def test_dedup_parity_and_probe(monkeypatch, dedup):
    monkeypatch.setenv("SERFSIM_DEDUP", dedup)
    L = lib()
    L.emu_probe.restype = C.c_ulong
    L.emu_probe_reset()
    n = 12_000
    P.run_against_oracle(emu_sim, E.leave_study(n, random_regular_graph(n, 16, 3), fanout=4, max_ticks=80))
    P.run_against_oracle(emu_sim, E.crash_study(n, random_regular_graph(n, 12, 4), fanout=4))
    skipped = L.emu_probe(22)
    assert (skipped > 0) == (dedup == "1"), skipped
