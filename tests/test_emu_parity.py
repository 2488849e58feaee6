"""Kernel logic on the CPU: the product's kernel sources, compiled for the host by tests/emu (every CUDA thread a fiber,
collectives honoured), against the oracle — the same comparisons as tests/test_gpu_parity.py at sizes a fiber
scheduler finishes in seconds.  This does not replace the GPU parity run (it cannot see memory-ordering, cache or
PTX-level behaviour); it catches indexing / control-flow / host-logic mistakes before GPU time is spent.
"""
import numpy as np
import pytest

import parity_lib as P
from emu_lib import emu_sim
from oracle_lib import oracle_sim
from serf_b200 import MemberStatus, scenarios


@pytest.mark.parametrize("seed", [1, 2])
def test_config0_full_mesh_256(seed):
    out = P.run_against_oracle(emu_sim, scenarios.full_mesh_leave(256, 3, seed))
    assert (out["member_status"][0][1:] == MemberStatus.LEFT).all()


def test_random_graph_single_slot():
    P.run_against_oracle(emu_sim, scenarios.random_graph_leave(6000, 16, 3, seed=1))


def test_random_graph_multi_slot_fanout4():
    P.run_against_oracle(emu_sim, scenarios.random_graph_leave(3000, 12, 4, seed=5, slots=4))


def test_fanout_eight():
    P.run_against_oracle(emu_sim, scenarios.random_graph_leave(2000, 12, 8, seed=3, slots=2))


def test_failure_detection():
    sc = scenarios.random_graph_fail(2500, 16, 3, seed=2)
    out = P.run_against_oracle(emu_sim, sc, suspicion_mult=2, suspicion_max_timeout_mult=2, probe_interval_ticks=2)
    assert (np.delete(out["member_status"][0], 5) == MemberStatus.FAILED).all()


def test_small_world_churn():
    sc = scenarios.small_world_churn(3000, 12, 0.1, 0.05, slots=4, window=30, seed=3)
    P.run_against_oracle(emu_sim, sc, suspicion_mult=2, suspicion_max_timeout_mult=2, probe_interval_ticks=2)


@pytest.mark.parametrize("seed", range(40))
def test_fuzz(seed):
    P.run_against_oracle(emu_sim, scenarios.fuzz(seed))


def test_compaction_path_is_taken_and_exact():
    """Unsaturated ticks of a trace-off run gather the active nodes of several tiles (SFS_PROBE 0..2 count the groups,
    the multi-tile groups and the groups needing more than one dense pass)."""
    import ctypes as C
    from emu_lib import lib
    L = lib()
    L.emu_probe.restype = C.c_ulong
    L.emu_probe_reset()
    P.run_against_oracle(emu_sim, scenarios.random_graph_leave(6000, 16, 3, seed=1), traces=(0,))
    assert L.emu_probe(0) > 0 and L.emu_probe(1) > 0 and L.emu_probe(2) > 0


def test_remove_failed_node_prune_reference_scenario():
    """serf_remove_failed_node_prune (serf/base/tests/serf/remove.rs:95-165): after the pruning force-leave the survivors no
    longer list the failed node (`wait_until_num_nodes(2, ..)` in the reference)."""
    for n in (3, 40):
        sc = scenarios.remove_failed_node_prune(n)
        out = P.run_against_oracle(emu_sim, sc)
        st = out["member_status"][0]
        assert (np.delete(st, 1) == MemberStatus.NONE).all(), st          # erased from every survivor's member table
        tr = out["trace"]
        assert tr["pending"][sc.ops[1][0] - 1] == 0                       # the failure had been detected and had settled before the prune


@pytest.mark.parametrize("seed", range(24))
def test_fuzz_prune(seed):
    P.run_against_oracle(emu_sim, scenarios.fuzz_prune(seed))


def test_sleeping_views_timer_wheel_and_idle_ticks(monkeypatch):
    """A crash with the memberlist LAN timers: the suspicion timers run for ~100 ticks in which nothing else happens.  Views that
    only wait for their timer sleep (SFS_PROBE 5 counts the views a visited node left asleep), their tiles are woken by the
    timer wheel (probe 4) and the ticks in which nothing can happen are skipped (probe 3) — with every trace row, `pending`
    included, the records and the clocks still equal to the oracle's, which visits every view in every tick."""
    import ctypes as C
    from emu_lib import lib
    L = lib()
    L.emu_probe.restype = C.c_ulong
    sc = scenarios.dissemination_storm(3000, 12, 3, slots=2, seed=3, with_fail=True)
    o = sc.build(oracle_sim, trace=1)
    to = o.run_until_converged(sc.max_ticks)
    ref = P.outputs(o, sc, to)
    assert to[0] > 60
    for trace, chunk in ((0, None), (1, None), (0, "4"), (1, "5")):
        L.emu_probe_reset()
        if chunk:
            monkeypatch.setenv("SERFSIM_CHUNK", chunk)     # small launch chunks: the host learns early that the cluster sleeps
        else:
            monkeypatch.delenv("SERFSIM_CHUNK", raising=False)
        f = sc.build(emu_sim, trace=trace)
        got = P.outputs(f, sc, f.run_until_converged(sc.max_ticks))
        # skipped on the device (launched before the host learnt that the cluster sleeps, probe 3) or not launched at all (probe 17)
        assert L.emu_probe(3) + L.emu_probe(17) > 20 and L.emu_probe(4) > 0, (L.emu_probe(3), L.emu_probe(17), L.emu_probe(4))
        if chunk:
            assert L.emu_probe(17) > 10
        if not trace:
            assert L.emu_probe(5) > 0
            assert L.emu_probe(20) > 0             # nodes of a due tile whose own deadline (node_due) lies later: no view visited
        P.assert_same(got, ref, with_hash=bool(trace), what=f"trace={trace} chunk={chunk}")
    # stepping one tick at a time takes the same decisions (the scheduler words live on the device, not in the call)
    f = sc.build(emu_sim, trace=1)
    for _ in range(to[0] + 1):
        f.step(1)
    o2 = sc.build(oracle_sim, trace=1)
    o2.step(to[0] + 1)
    P.assert_same(P.outputs(f, sc, None), P.outputs(o2, sc, None), with_hash=True)


@pytest.mark.parametrize("ahead", ["0", "2"])
def test_multi_slot_requests_one_tile_ahead(ahead, monkeypatch):
    """Multi-slot runs request node word, gossip peers and the probable first view's record one tile ahead in saturated ticks
    (SERFSIM_AHEAD, tick_kernel.cu `Ahead`); 2 forces the path in every tick of the tile walk, 0 switches it off.  Probe 19 counts the
    nodes requested ahead, probe 18 the records that were used (the guess of the first view was right)."""
    import ctypes as C
    from emu_lib import lib
    L = lib()
    L.emu_probe.restype = C.c_ulong
    monkeypatch.setenv("SERFSIM_AHEAD", ahead)
    monkeypatch.setenv("SERFSIM_COMPACT", "0")             # every tick walks its tiles
    L.emu_probe_reset()
    for sc in (scenarios.dissemination_storm(3000, 12, 3, slots=2, seed=3, with_fail=True), scenarios.random_graph_leave(5000, 16, 4, seed=2, slots=3),
               scenarios.fuzz(3), scenarios.fuzz(11), scenarios.fuzz_prune(5)):
        P.run_against_oracle(emu_sim, sc)
    if ahead == "2":
        assert L.emu_probe(19) > 1000 and L.emu_probe(18) > 100, (L.emu_probe(19), L.emu_probe(18))
    else:
        assert L.emu_probe(19) == 0


@pytest.mark.parametrize("mode", ["0", "1", "2"])
def test_single_view_ticks(mode, monkeypatch):
    """Multi-slot runs in production mode, exactly one subject ever down: ticks in which only that subject's view has business run the
    single-slot kernel on it (SERFSIM_SV=1: both kernels launched, the device picks; probe 21 counts the CTAs of single-view kernels
    that ran).  SERFSIM_SV=2 runs the general kernel alone and fails with error 4 if a view outside a one-element set had business;
    0 switches the dispatch off.  All three equal the oracle."""
    import ctypes as C
    from emu_lib import lib
    L = lib()
    L.emu_probe.restype = C.c_ulong
    monkeypatch.setenv("SERFSIM_SV", mode)
    L.emu_probe_reset()
    scs = [scenarios.dissemination_storm(3000, 12, 3, slots=2, seed=3, with_fail=True), scenarios.dissemination_storm(2500, 10, 4, slots=3, seed=5, with_fail=True)]
    scs += [scenarios.fuzz(k) for k in range(12)] + [scenarios.fuzz_prune(k) for k in range(6)]
    for sc in scs:
        P.run_against_oracle(emu_sim, sc, traces=(0,))
    if mode == "1":
        assert L.emu_probe(21) > 20, L.emu_probe(21)
    else:
        assert L.emu_probe(21) == 0


def test_config1_shape_100k_nodes():
    """BASELINE configs[1] at full size (100 K-node random graph, fan-out 3) through the host-compiled kernels:
    391 tiles over 4 CTAs, dense and sparse ticks, production mode (trace off)."""
    P.run_against_oracle(emu_sim, scenarios.random_graph_leave(100_000, 16, 3, seed=1), traces=(0,))


def test_config2_shape_small_world_churn_100k():
    """BASELINE configs[2] shape (small world, 5 % of the nodes crash / return, 8 tracked subjects, probing on) at
    100 K nodes, production mode."""
    sc = scenarios.small_world_churn(100_000, 16, 0.1, 0.05, slots=8, window=60, seed=3)
    P.run_against_oracle(emu_sim, sc, traces=(0,), suspicion_mult=2, suspicion_max_timeout_mult=2, probe_interval_ticks=2)


@pytest.mark.parametrize("seed", range(30))
def test_fuzz_with_user_events_and_injectors(seed):
    """Every operation kind, reaper, probing, tracked user events (with aliases) and byzantine injectors at once."""
    sc = scenarios.fuzz_features(seed)
    sc.max_ticks = 1200                    # injector runs with push-pull / reaper rounds may never go quiet: both sides stop at the cap
    P.run_against_oracle(emu_sim, sc)


@pytest.mark.skipif(not __import__("os").environ.get("SERFSIM_SLOW"), reason="≈ 2 min and 3 GB: set SERFSIM_SLOW=1")
def test_bench_workload_full_10m_nodes():
    """The bench workload itself — BASELINE configs[3] shape on one device: 10 M-node random graph, fan-out 4, one
    dissemination to quiescence — through the host-compiled kernel in production mode, against the oracle (8 threads)."""
    from oracle_lib import lib as olib
    sc = scenarios.dissemination_storm(10_000_000, 16, 4, slots=1, seed=1)
    f = sc.build(emu_sim, trace=0)
    tf = f.run_until_converged(sc.max_ticks)
    o = sc.build(oracle_sim, trace=0)
    olib().oracle_sim_set_threads(o._h, 8)
    o.reset(sc.cfg["seed"])
    sc.schedule(o)
    P.assert_same(P.outputs(f, sc, tf), P.outputs(o, sc, o.run_until_converged(sc.max_ticks)), with_hash=False)
