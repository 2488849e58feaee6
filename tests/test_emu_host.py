"""Host-side logic of the C ABI (serf_b200/csrc/serfsim.cu) exercised on the CPU through the host-compiled build of
tests/emu: stepping API, convergence loop variants, event callback, timing hooks, validation.  Results are compared
with the oracle where there is something to compare."""
import ctypes as C

import numpy as np
import pytest

import parity_lib as P
from emu_lib import emu_sim, lib
from oracle_lib import oracle_sim
from serf_b200 import MemberStatus, scenarios
from serf_b200.sim import Config, Op, SerfsimError


def test_step_by_step_equals_run_until_converged():
    sc = scenarios.random_graph_leave(2000, 12, 3, seed=2, slots=2)
    o = sc.build(oracle_sim, trace=1)
    to, ok = o.run_until_converged(sc.max_ticks)
    ref = P.outputs(o, sc, None)
    g = sc.build(emu_sim, trace=1)
    for _ in range(to + 1):
        g.step(1)
    P.assert_same(P.outputs(g, sc, None), ref, with_hash=True)
    h = sc.build(emu_sim, trace=0)
    h.step(5)
    h.step(to + 1 - 5)
    P.assert_same(P.outputs(h, sc, None), ref, with_hash=False)


def test_max_ticks_reached_returns_not_converged():
    sc = scenarios.random_graph_leave(2000, 12, 3, seed=2)
    g, o = sc.build(emu_sim, trace=1), sc.build(oracle_sim, trace=1)
    assert g.run_until_converged(6) == o.run_until_converged(6) == (6, False)
    tg, to = g.run_until_converged(sc.max_ticks), o.run_until_converged(sc.max_ticks)      # and both continue from there
    P.assert_same(P.outputs(g, sc, tg), P.outputs(o, sc, to), with_hash=True)


def test_long_run_grows_the_trace_buffer():
    """More than 1024 ticks: the device trace / kind-counter arrays are reallocated and copied."""
    sc = scenarios.random_graph_leave(600, 8, 3, seed=1)
    g, o = sc.build(emu_sim, trace=1), sc.build(oracle_sim, trace=1)
    g.run_until_converged(sc.max_ticks), o.run_until_converged(sc.max_ticks)
    g.inject(1500, Op.JOIN, int(sc.subjects[0]), 0)
    o.inject(1500, Op.JOIN, int(sc.subjects[0]), 0)
    tg, to = g.run_until_converged(4000), o.run_until_converged(4000)
    assert g.stats()["tick"] > 1500
    P.assert_same(P.outputs(g, sc, tg), P.outputs(o, sc, to), with_hash=True)


def test_launch_chunks_1_4_16_give_the_same_result(monkeypatch):
    sc = scenarios.random_graph_leave(3000, 12, 4, seed=3)
    o = sc.build(oracle_sim, trace=1)
    ref = P.outputs(o, sc, o.run_until_converged(sc.max_ticks))
    for chunk in ("1", "4", "16"):
        monkeypatch.setenv("SERFSIM_CHUNK", chunk)
        g = sc.build(emu_sim, trace=0)
        P.assert_same(P.outputs(g, sc, g.run_until_converged(sc.max_ticks)), ref, with_hash=False, what=f"chunk {chunk}")
    g = sc.build(emu_sim, trace=0)
    assert g.run_until_converged(7) == (7, False)


@pytest.mark.parametrize("chunk", ["1", "3", "9"])
def test_chunk_size_does_not_change_results(monkeypatch, chunk):
    monkeypatch.setenv("SERFSIM_CHUNK", chunk)
    P.run_against_oracle(emu_sim, scenarios.fuzz(11), traces=(0,))                # has reaper / push-pull boundary ticks


def test_event_callback_reports_agreed_status_changes():
    sc = scenarios.random_graph_fail(1500, 16, 3, seed=2)            # subject 5 crashes, subject n/2 leaves
    g = sc.build(emu_sim, trace=0, suspicion_mult=2, suspicion_max_timeout_mult=2, probe_interval_ticks=2)
    seen = []
    g.set_event_callback(lambda tick, ty, ids: seen.append((ty, tuple(ids))))
    g.run_until_converged(sc.max_ticks)
    kinds = {ty for ty, _ in seen}
    assert 2 in kinds and 1 in kinds                                  # MemberEventType::Failed and ::Leave (event.rs:325-328)
    assert (2, (5,)) in seen and (1, (750,)) in seen
    n = len(seen)
    g.step(3)                                                         # nothing new: no repeated reports
    assert len(seen) == n


def test_timing_hooks():
    sc = scenarios.random_graph_leave(1000, 8, 3, seed=1)
    g = sc.build(emu_sim)
    g.set_tick_timing(True)
    t, ok = g.run_until_converged(sc.max_ticks)
    ms = g.tick_times_ms()
    assert len(ms) == t + 1 and (ms >= 0).all()
    dev_ms, launches = g.last_step_device_ms()
    assert launches >= t + 1 and dev_ms >= 0
    g2 = sc.build(emu_sim)
    g2.run_until_converged(sc.max_ticks)
    with pytest.raises(SerfsimError):
        g2.tick_times_ms(0, 3)                                        # timing was not enabled


def test_create_and_inject_validation():
    L = lib()
    cfg = Config()
    L.serfsim_default_config(C.byref(cfg))
    assert (cfg.fanout, cfg.retransmit_mult, cfg.suspicion_mult, cfg.suspicion_max_timeout_mult, cfg.probe_interval_ticks) == (3, 4, 4, 6, 5)
    assert cfg.abi_version == L.serfsim_abi_version()
    for bad in (dict(fanout=0), dict(fanout=9)):
        with pytest.raises(SerfsimError):
            emu_sim(100, 1, **bad)
    with pytest.raises(SerfsimError):
        emu_sim(100, 17)
    g = emu_sim(100, 1)
    with pytest.raises(SerfsimError):
        g.step(1)                                                     # no topology yet
    sc = scenarios.random_graph_leave(300, 8, 3, seed=1)
    g = sc.build(emu_sim)
    with pytest.raises(SerfsimError):
        g.inject(0, Op.LEAVE, 17, 0)                                  # join/leave origin must be a tracked subject
    with pytest.raises(SerfsimError):
        g.inject(0, Op.FAIL, int(sc.subjects[0]), 0)                  # one operation per node per tick (a LEAVE is scheduled there)
    g.step(2)
    with pytest.raises(SerfsimError):
        g.inject(1, Op.FAIL, 9, 0)                                    # in the past
    assert g.shard_range() == (0, 300) if hasattr(g, "shard_range") else True


def test_cpp_host_layer_end_to_end(tmp_path):
    """include/serfsim.hpp (the C++ host layer with the reference's names) driving the host-compiled library: the
    configs[0] leave scenario with the event callback, then two user events — the program tests/test_abi.py runs on a
    GPU box, here linked against the emulated build."""
    import os
    import subprocess
    from emu_lib import build
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    so = build()
    exe = str(tmp_path / "host_layer_check")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I" + os.path.join(root, "include"), os.path.join(root, "tests", "cpp", "host_layer_check.cpp"),
                           so, "-Wl,-rpath," + os.path.dirname(so), "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "left=255 leave_events=1" in r.stdout and "seen=256/256 delivered=512" in r.stdout


def test_graft_entry_smoke_logic_runs(monkeypatch):
    """__graft_entry__.smoke() (the driver's first GPU check) with the library swapped for the host-compiled build: the
    Python side of the smoke test itself is exercised here, so a typo cannot be what fails on the GPU box."""
    import os
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    import __graft_entry__ as ge
    from serf_b200 import sim
    monkeypatch.setattr(sim, "_LIB", lib())
    ge.smoke()


@pytest.mark.parametrize("seed", range(1, 9))
@pytest.mark.parametrize("chunk", ["4", "3"])
def test_multi_phase_production_mode_rewind(monkeypatch, seed, chunk):
    """trace=0 (tile skipping, lazy loads, compaction): converge → inject at the CURRENT tick → continue.  The convergence
    loop rewinds the ticks it launched past the quiescent one; the hot-tile flags are double-buffered by tick parity, so
    an odd rewind used to leave the watcher tiles unscheduled for the next tick (their SWIM probe of that tick was lost)."""
    monkeypatch.setenv("SERFSIM_CHUNK", chunk)
    n = 1500
    sc = scenarios.random_graph_leave(n, 12, 3, seed=seed, slots=2, graph_seed=seed + 20)
    cfg = dict(suspicion_mult=2, suspicion_max_timeout_mult=2, probe_interval_ticks=2)
    sc.ops = [(0, Op.JOIN, int(sc.subjects[0]), 0)]
    g, o = sc.build(emu_sim, trace=0, **cfg), sc.build(oracle_sim, trace=1, **cfg)
    assert g.run_until_converged(sc.max_ticks) == o.run_until_converged(sc.max_ticks)
    for sim in (g, o):
        sim.inject(sim.stats()["tick"], Op.FAIL, int(sc.subjects[1]), 0)
    tg, to = g.run_until_converged(5000), o.run_until_converged(5000)
    P.assert_same(P.outputs(g, sc, tg), P.outputs(o, sc, to), with_hash=False)
    for sim in (g, o):                                               # and once more: the subject returns, a force-leave follows later
        t = sim.stats()["tick"]
        sim.inject(t, Op.REJOIN, int(sc.subjects[1]), 0)
        sim.inject(t + 3, Op.FORCE_LEAVE, 7, 0)
    tg, to = g.run_until_converged(5000), o.run_until_converged(5000)
    P.assert_same(P.outputs(g, sc, tg), P.outputs(o, sc, to), with_hash=False)


def test_results_async_returns_the_getters_values():
    """serfsim_results_async / _wait (ABI v4): the three result vectors of a slot through the staging ring, several calls in
    flight (more than the ring holds), partial requests (NULL pointers)."""
    sc = scenarios.random_graph_leave(3000, 12, 3, seed=2, slots=3)
    g = sc.build(emu_sim, trace=0)
    g.run_until_converged(sc.max_ticks)
    bufs = []
    for rep in range(2):
        for s in range(3):
            st, lt, ck = np.zeros(g.count, np.uint8), np.zeros(g.count, np.uint32), np.zeros(g.count, np.uint32)
            n = g.results_async(s, status=st, status_ltime=lt, lamport=ck if s == 0 else None)
            assert n == g.count * (1 + 4 + (4 if s == 0 else 0))
            bufs.append((s, st, lt, ck))
    g.results_wait()
    for s, st, lt, ck in bufs:
        assert (st == g.member_status(s)).all() and (lt == g.status_ltime_u32(s)).all()
        if s == 0:
            assert (ck == g.lamport_time_u32()).all()


def test_jump_after_a_probe_tick_with_a_host_operation():
    """The host jumps over a sleeping stretch after ONE single-tick launch whose gate has judged the row before it.  If that probe tick
    carries a host operation (here one that changes nothing), its own row is new and unjudged: the jump must wait for one more single tick.
    Fuzz scenario 16 with the default launch chunks (8, 16, 32, 32 → the chunk ends on tick 87, the no-op operation sits at tick 88, the
    reaper at 99): the run was reported quiescent at tick 98 instead of 88."""
    sc = scenarios.fuzz(16)
    sc.max_ticks = 1500
    o = sc.build(oracle_sim, trace=1)
    to = o.run_until_converged(sc.max_ticks)
    for trace in (1, 0):
        g = sc.build(emu_sim, trace=trace)
        assert g.run_until_converged(sc.max_ticks) == to


@pytest.mark.parametrize("seed", range(1000, 1012))
def test_late_operations_in_sleeping_stretches(seed, monkeypatch):
    """Fuzz scenarios with extra (mostly no-op) host operations scattered over the 300 ticks after the busy part — the convergence loop's
    probe / jump / gate rules with the default launch chunks, in trace mode, and with a small fixed chunk (a sample of
    tools/campaigns/late_ops.py)."""
    import importlib.util
    import os
    spec = importlib.util.spec_from_file_location("late_ops_gen", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "campaigns", "late_ops_gen.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    sc = gen.late(seed)
    o = sc.build(oracle_sim, trace=1)
    ref = P.outputs(o, sc, o.run_until_converged(sc.max_ticks))
    for trace, chunk in ((0, None), (1, None), (0, str(2 + seed % 11))):
        if chunk:
            monkeypatch.setenv("SERFSIM_CHUNK", chunk)
        else:
            monkeypatch.delenv("SERFSIM_CHUNK", raising=False)
        g = sc.build(emu_sim, trace=trace)
        P.assert_same(P.outputs(g, sc, g.run_until_converged(sc.max_ticks)), ref, with_hash=bool(trace), what=f"trace={trace} chunk={chunk}")
