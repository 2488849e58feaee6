"""Per-view passes choose their loads from their own view's traffic (host build of the kernels, tests/emu).

A pass streams an inbox plane only if its view sent that kind in the previous tick, and it requests every node up front only if its
view's own messages saturated that tick (DESIGN §5, "Per-view passes").  Both only choose what a pass loads, so every trace row, record,
clock and the state hash must equal the oracle's.  The per-view counters are trusted only after a tick whose inbox writes all came
from passes; after a tick of the general kernel (host operation, reaper round) the passes fall back to the whole tick's counters.

Coverage probes of the host build: 23 = a pass used the whole-tick fallback, 24 = a pass took the compacted walk in a tick the
whole-tick counters call saturated, 25 = a pass left unread the plane of a kind that was in flight in another view.
"""
import ctypes as C

import numpy as np
import pytest

import parity_lib as P
from emu_lib import emu_sim, lib
from oracle_lib import oracle_sim
from serf_b200 import Op, scenarios


def _probes():
    L = lib()
    L.emu_probe.restype = C.c_ulong
    return L


def leave_fail_study():
    """The bench study's shape (one leave and one crash at tick 0, memberlist LAN timers) at 3000 nodes."""
    return scenarios.dissemination_storm(3000, 12, 4, slots=2, seed=3, with_fail=True)


def offset_storm():
    """Three views whose waves are offset by host operations: a leave at tick 0, a crash at tick 6, a second leave at tick 12."""
    sc = scenarios.dissemination_storm(3000, 12, 4, slots=3, seed=5)
    s = [int(x) for x in sc.subjects]
    sc.ops = [(0, Op.LEAVE, s[0], 0), (6, Op.FAIL, s[1], 0), (12, Op.LEAVE, s[2], 0)]
    return sc


@pytest.mark.parametrize("compact", ["1", "0"])
@pytest.mark.parametrize("make", [leave_fail_study, offset_storm])
def test_passes_decide_from_their_own_view_and_stay_exact(make, compact, monkeypatch):
    monkeypatch.setenv("SERFSIM_COMPACT", compact)
    L = _probes()
    sc = make()
    o = sc.build(oracle_sim, trace=1)
    to = o.run_until_converged(sc.max_ticks)
    L.emu_probe_reset()
    f = sc.build(emu_sim, trace=0)
    P.assert_same(P.outputs(f, sc, f.run_until_converged(sc.max_ticks)), P.outputs(o, sc, to), with_hash=False)
    # The per-view counters add up to the whole tick's message count in every tick that ran as passes.
    vk = f.tick_view_kinds()
    msgs = f.tick_trace()["messages"]
    ran = vk.reshape(len(vk), -1).sum(axis=1) > 0
    assert ran.sum() > 5
    assert (vk.sum(axis=(1, 2))[ran] == msgs[ran]).all()
    assert L.emu_probe(25) > 0, "no pass skipped a plane of a kind that was in flight in another view"
    if compact == "1":
        assert L.emu_probe(24) > 0, "no pass took the compacted walk in a tick another view saturated"
    else:
        assert L.emu_probe(24) == 0


def test_after_a_general_kernel_tick_passes_fall_back_to_whole_tick_counters():
    """Stepping one tick at a time: the passes of the tick after a host operation or a reaper round use the whole tick's counters,
    those after a tick of passes their own view's."""
    L = _probes()
    sc = offset_storm()
    cfg = dict(reap_interval_ticks=9, tombstone_timeout_ticks=400, reconnect_timeout_ticks=400)
    o = sc.build(oracle_sim, trace=1, **cfg)
    f = sc.build(emu_sim, trace=0, **cfg)
    op_ticks = {t for (t, _, _, _) in sc.ops}
    general = lambda t: t in op_ticks or (t + 1) % 9 == 0          # ticks the general kernel runs
    fell_back = {}
    for t in range(30):
        before = L.emu_probe(23)
        f.step(1)
        fell_back[t] = L.emu_probe(23) - before
    o.step(30)
    P.assert_same(P.outputs(f, sc, None), P.outputs(o, sc, None), with_hash=False)
    for t in range(1, 30):
        if general(t):
            assert fell_back[t] == 0                                # not a pass tick at all
        elif general(t - 1):
            assert fell_back[t] > 0, t
        else:
            assert fell_back[t] == 0, t
    assert sum(1 for t in range(1, 30) if not general(t) and general(t - 1) and fell_back[t]) >= 4
    vk = f.tick_view_kinds()
    assert not vk[[t for t in range(30) if general(t)]].any()        # the general kernel leaves no per-view counts
    assert np.asarray(vk).sum() > 0
