"""Sharded path logic on the CPU: W ranks as threads of this process, each driving its own handle of the
host-compiled kernels (tests/emu); the "NVLink windows" are plain shared memory with real acquire/release on the
flags, the host collectives (barrier, u64 all-reduce) are thread primitives.  Concatenated records and the
all-reduced trace must equal the single oracle's — the comparisons of tests/test_gpu_multi.py at small sizes."""
import pytest

import parity_lib as P
from emu_lib import emu_sim
from serf_b200 import scenarios


@pytest.mark.parametrize("world", [2, 3, 4])
def test_sharded_random_graph(world):
    P.run_against_oracle(emu_sim, scenarios.random_graph_leave(3001, 12, 3, seed=2, slots=1), world=world)


@pytest.mark.parametrize("world", [2, 4])
def test_sharded_multi_slot_fanout4(world):
    P.run_against_oracle(emu_sim, scenarios.random_graph_leave(2500, 12, 4, seed=3, slots=3), world=world)


# One node per shard: the reciprocal that maps a target to its shard has no exact u32 value for shard_size 1
@pytest.mark.parametrize("n,world", [(3, 3), (4, 4), (8, 8)])
def test_sharded_one_node_per_shard(n, world):
    P.run_against_oracle(emu_sim, scenarios.full_mesh_leave(n, 3, 1), world=world)


def test_sharded_failure_detection():
    P.run_against_oracle(emu_sim, scenarios.random_graph_fail(2000, 16, 3, seed=2), world=2, suspicion_mult=2, suspicion_max_timeout_mult=2, probe_interval_ticks=2)


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_cluster_sleeps_through_the_suspicion_timers(world, monkeypatch):
    """LAN timers: ~30 ticks in which every shard only waits for suspicion deadlines.  The ranks publish their scheduler verdicts
    with their rows, every rank derives the same "sleep until" tick, and the hosts do not launch those ticks (probe 17 counts
    them) — rows, records and clocks still equal the oracle's."""
    import ctypes as C
    from emu_lib import lib
    L = lib()
    L.emu_probe.restype = C.c_ulong
    L.emu_probe_reset()
    monkeypatch.setenv("SERFSIM_CHUNK", "4")
    P.run_against_oracle(emu_sim, scenarios.dissemination_storm(3000, 12, 3, slots=2, seed=3, with_fail=True), world=world)
    assert L.emu_probe(17) > 20 * world            # both trace modes, every rank


@pytest.mark.parametrize("seed", [7, 9, 12])
def test_sharded_fuzz(seed):
    P.run_against_oracle(emu_sim, scenarios.fuzz(seed, n=600, slots=4), world=2, push_pull_interval_ticks=0)


# ---- user events across shards: remote targets get kind-3 window entries (event bit + the origin's Lamport time) ----
@pytest.mark.parametrize("world", [2, 3])
def test_sharded_user_events(world):
    P.run_against_oracle(emu_sim, scenarios.user_event_storm(2501, 12, 3, seed=3, n_events=5, spacing=2, churn=30, with_leave=True), world=world)


def test_sharded_user_events_aliased_fanout4():
    P.run_against_oracle(emu_sim, scenarios.user_event_storm(2000, 12, 4, seed=5, n_events=3, spacing=2, alias=True), world=4)


# ---- push-pull rounds across shards: partners on other ranks are read through the peer mapping of their snapshot ----
@pytest.mark.parametrize("world,pp", [(2, 7), (3, 5), (4, 16)])
def test_sharded_push_pull(world, pp):
    from serf_b200 import small_world_graph
    n = 1500
    sc = scenarios.Scenario("pp", n, 2, small_world_graph(n, 8, 0.1, 5), [3, n // 2],
                            [(0, scenarios.Op.LEAVE, 3, 0), (1, scenarios.Op.FAIL, n // 2, 0), (40, scenarios.Op.REJOIN, n // 2, 0)],
                            dict(fanout=3, seed=4, retransmit_mult=1, suspicion_mult=2, suspicion_max_timeout_mult=2, probe_interval_ticks=2),
                            max_ticks=3000)
    P.run_against_oracle(emu_sim, sc, world=world, push_pull_interval_ticks=pp)


@pytest.mark.parametrize("seed", [3, 5, 11])
def test_sharded_fuzz_with_push_pull_and_reaper(seed):
    P.run_against_oracle(emu_sim, scenarios.fuzz(seed, n=500, slots=3), world=2)


# ---- byzantine injectors across shards: triples in the peer's window, verdict by the receiving shard's drain kernel ----
@pytest.mark.parametrize("world", [2, 4])
def test_sharded_byzantine(world):
    P.run_against_oracle(emu_sim, scenarios.byzantine_injectors(2400, 16, 4, 0.02, seed=1), world=world)


def test_sharded_byzantine_heavy_three_ranks():
    P.run_against_oracle(emu_sim, scenarios.byzantine_injectors(1501, 12, 3, 0.2, seed=3), world=3)


def test_sharded_stage_overflow_path():
    """8 subjects × fan-out 8: a tile produces far more cross-shard entries than the shared-memory stage holds
    (3072 per CTA), so the write-through path behind the stage is taken — results unchanged."""
    P.run_against_oracle(emu_sim, scenarios.random_graph_leave(1500, 12, 8, seed=6, slots=8), world=2)


def test_window_overflow_is_reported(monkeypatch):
    """A receive window too small for the traffic must fail loudly (SERFSIM_E_COMM), never drop entries silently."""
    from serf_b200.sim import SerfsimError
    monkeypatch.setenv("SERFSIM_WIN_FACTOR", "0.0001")
    sc = scenarios.random_graph_leave(30000, 12, 8, seed=6, slots=8)
    with pytest.raises(SerfsimError) as ei:
        P.run_ranks(sc, 2, 0)
    assert ei.value.code == -6


@pytest.mark.parametrize("seed", [1, 4, 6, 8, 13, 21, 131, 163, 325])
def test_sharded_fuzz_with_user_events_and_injectors(seed):
    """fuzz_features across 2–4 ranks: operations, reaper, probing, push-pull, user events and injectors, all crossing shards.
    (131 / 163 / 325: push-pull rounds whose partner holds an event the puller's shard has not received yet — a randomized
    campaign over 300 such scenarios found that the replay then lacked the event's Lamport time.)"""
    sc = scenarios.fuzz_features(seed, n=(400 + 37 * seed) if seed < 100 else 300 + 13 * (seed % 40), slots=3 if seed < 100 else 1 + seed % 4)
    sc.max_ticks = 400 if seed < 100 else 300   # some injector runs never go quiet (reaper ticks keep merging): both sides stop at the cap
    world = (2 + seed % 2) if seed < 100 else 2 + seed % 3
    P.run_against_oracle(emu_sim, sc, world=world)


def test_sharded_user_events_need_bigger_windows():
    """5 events × fan-out 3 from every node: more cross-shard entries per tick than the windows serfsim_create sizes for
    membership traffic alone — serfsim_set_user_events must have resized them (it used to overflow at this size)."""
    P.run_against_oracle(emu_sim, scenarios.user_event_storm(20_000, 16, 3, seed=3, n_events=5, spacing=2, churn=50, with_leave=True), world=2)


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_user_events_with_push_pull(world):
    """Event replay of a push-pull round when the partner lives in another shard (its event snapshot is peer-mapped)."""
    P.run_against_oracle(emu_sim, scenarios.user_event_storm(2001, 8, 2, seed=6, n_events=5, spacing=2, churn=30, with_leave=True), world=world, push_pull_interval_ticks=5, retransmit_mult=1)


def test_sharded_byzantine_with_push_pull():
    P.run_against_oracle(emu_sim, scenarios.byzantine_injectors(2400, 12, 3, 0.05, seed=5), world=3, push_pull_interval_ticks=6)


def test_sharded_handle_without_hooks_or_connection():
    """A world-2 handle whose host never installed the collective hooks: every call that needs a barrier or an all-reduce fails
    with SERFSIM_E_COMM instead of returning a shard-local answer, and a step fails because the handle is not connected.  A run of
    zero ticks launches nothing and reports "not converged at tick 0", user events or not.  Once the handle is connected, user
    events that need bigger receive windows are refused (the windows were exported already)."""
    from serf_b200.sim import SerfsimError
    E_INVAL, E_COMM = -1, -6

    def error(f, *args):
        with pytest.raises(SerfsimError) as ei:
            f(*args)
        return ei.value

    def code(f, *args):
        return error(f, *args).code

    sc = scenarios.random_graph_leave(600, 8, 3, seed=2, slots=1)

    def handle():
        g = emu_sim(sc.n, sc.slots, rank=0, world_size=2, **sc.cfg)
        g.set_topology(sc.row_ptr, sc.col)
        return g

    g = handle()
    g.set_user_events([1, 2])
    g.set_byzantine([1, 400])
    assert code(g.state_hash) == E_COMM
    assert code(g.user_event_stats) == E_COMM
    assert code(g.user_event_ltime, 0) == E_COMM
    assert code(g.anomaly_flags) == E_COMM
    assert code(g.byzantine_stats) == E_COMM
    assert code(g.step, 1) == E_COMM
    assert g.run_until_converged(0) == (0, False)
    g.close()

    g = handle()
    g.connect_loopback()
    e = error(g.set_user_events, [1, 2, 3])
    assert e.code == E_INVAL and "resizes the receive windows" in str(e), str(e)
    g.close()


def test_loopback_profiling_aid_runs():
    """serfsim_comm_loopback: a world-4 handle exchanging with itself (tools/loopback_profile.py).  Its results are meaningless by
    construction; what is checked is that the sharded kernels run to quiescence through the windows without an error."""
    sc = scenarios.random_graph_leave(4000, 12, 3, seed=2, slots=1)
    g = sc.build(emu_sim, rank=0, world_size=4, trace=0)
    g.connect_loopback()
    ticks, ok = g.run_until_converged(400)
    assert ok and g.stats()["edge_updates"] > 0
