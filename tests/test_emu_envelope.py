"""The edges of the ABI's input range on the host build of the kernels (tests/emu) against the oracle: CSR topologies whose
out-degrees differ (the general row-offset path, isolated nodes, hubs, self-loops, duplicate edges), fan-out 6–8 with 9–16
slots (the per-view passes), the scheduler switches SERFSIM_NO_SKIP / SERFSIM_NO_JUMP, sharded runs whose shards differ in
having a uniform degree, and the ABI's limits on degree, fan-out and slots.  The host build runs 12 CTAs of the single-slot
kernel at most (one "SM" by default: 3 CTAs × 2), so every CTA owns many tiles at these sizes; SFS_PROBE counters prove that
the targeted paths ran.  tests/test_gpu_z_envelope.py runs the same inputs on the device."""
import ctypes as C

import numpy as np
import pytest

import envelope_lib as E
import parity_lib as P
from emu_lib import emu_sim, lib
from serf_b200 import SerfsimError
from serf_b200.sim import random_regular_graph


def probes():
    L = lib()
    L.emu_probe.restype = C.c_ulong
    return L


# ---- irregular CSR -------------------------------------------------------------------------------------------
def test_each_handle_reads_its_own_switches(capfd):
    """The run-time switches are read when a handle is created: in one process, a handle under SERFSIM_GRIDMUL=1 gets one wave of
    CTAs and the next one, without it, two."""
    n = 64 * E.TILE
    one = E.grid_for(emu_sim, n, capfd, {"SERFSIM_GRIDMUL": "1", "SERFSIM_EMU_SMS": "4"})
    two = E.grid_for(emu_sim, n, capfd, {"SERFSIM_EMU_SMS": "4"})
    assert one[1] == 4 * 3 and two == (one[0], 2 * one[1]), (one, two)


def test_irregular_graph_shape():
    rp, col = E.irregular_graph(20_000, 1, self_loops=0.05, duplicates=0.05)
    deg = np.diff(rp.astype(np.int64))
    assert (deg == 0).mean() > 0.03 and ((deg > 0) & (deg < 3)).mean() > 0.1 and (deg > 8).any() and deg.max() >= 1000
    src = np.repeat(np.arange(20_000), deg)
    assert (col == src).any()                                                  # self-loops
    same_as_prev = np.zeros(col.size, bool)
    same_as_prev[1:] = (col[1:] == col[:-1]) & (src[1:] == src[:-1])
    assert same_as_prev.sum() > 1000                                           # duplicate edges
    assert E.envelope_fuzz(5).name == E.envelope_fuzz(5).name and (E.envelope_fuzz(5).col == E.envelope_fuzz(5).col).all()


def test_irregular_leave_and_lan_crash_multi_tile():
    """12 K nodes on 6 CTAs: 8 tiles per CTA.  Leaves on an irregular graph (both trace modes) and a crash with the LAN timers in
    production mode: compaction groups of several tiles, groups needing more than one dense pass, the timer wheel and sleeping
    nodes of due tiles.  (The crash runs on a regular graph: isolated nodes holding mail would keep every tile awake.)"""
    L = probes()
    n = 12_000
    topo = E.irregular_graph(n, 3)
    assert np.diff(topo[0].astype(np.int64)).min() == 0
    P.run_against_oracle(emu_sim, E.leave_study(n, topo, fanout=4, max_ticks=80))
    L.emu_probe_reset()
    P.run_against_oracle(emu_sim, E.leave_study(n, topo, fanout=3, seed=5, max_ticks=80), traces=(0,))
    P.run_against_oracle(emu_sim, E.crash_study(n, random_regular_graph(n, 12, 4), fanout=4), traces=(0,))
    assert L.emu_probe(0) > 0 and L.emu_probe(1) > 0 and L.emu_probe(2) > 0, [L.emu_probe(i) for i in range(3)]
    assert L.emu_probe(4) > 0 and L.emu_probe(20) > 0, (L.emu_probe(4), L.emu_probe(20))


def test_irregular_crash_short_timers_self_loops_duplicates():
    topo = E.irregular_graph(6000, 4, self_loops=0.05, duplicates=0.05)
    P.run_against_oracle(emu_sim, E.crash_study(6000, topo, fanout=3, short_timers=True, max_ticks=120))


@pytest.mark.parametrize("seed", range(12))
def test_irregular_fuzz(seed):
    P.run_against_oracle(emu_sim, E.envelope_fuzz(seed, topology="irregular"))


def test_uniform_graph_general_path(monkeypatch):
    """SERFSIM_UDEG=0: a uniform graph through the general (row_ptr) path gives what the arithmetic row offsets give."""
    sc = E.leave_study(8000, random_regular_graph(8000, 12, 9), fanout=4)
    a = P.run_against_oracle(emu_sim, sc, traces=(0,))
    monkeypatch.setenv("SERFSIM_UDEG", "0")
    P.assert_same(P.run_against_oracle(emu_sim, sc, traces=(0,)), a, with_hash=True)


# ---- fan-out 6–8 × slots 9–16 --------------------------------------------------------------------------------
def wide_fuzz_seeds(k):
    """The first k seeds whose envelope_fuzz scenario has fan-out ≥ 6 and at least 9 slots."""
    out, s = [], 0
    while len(out) < k:
        sc = E.envelope_fuzz(s)
        if sc.cfg["fanout"] >= 6 and sc.slots >= 9:
            out.append(s)
        s += 1
    return out


@pytest.mark.parametrize("sv", ["0", "1"])
def test_fanout8_slots12_storm(sv, monkeypatch):
    """A crash + leave storm, 12 slots, fan-out 8; SERFSIM_SV=1 runs the production ticks as per-view passes (probe 21)."""
    L = probes()
    monkeypatch.setenv("SERFSIM_SV", sv)
    L.emu_probe_reset()
    sc = E.crash_and_leave_study(3000, random_regular_graph(3000, 12, 7), fanout=8, slots=12)
    P.run_against_oracle(emu_sim, sc)
    assert (L.emu_probe(21) > 20) == (sv == "1"), L.emu_probe(21)


@pytest.mark.parametrize("seed", wide_fuzz_seeds(8))
def test_wide_fuzz(seed):
    sc = E.envelope_fuzz(seed)
    assert sc.cfg["fanout"] >= 6 and sc.slots >= 9
    P.run_against_oracle(emu_sim, sc)


def test_fuzz_draws_the_whole_range():
    scs = [E.envelope_fuzz(s) for s in range(200)]
    assert {sc.cfg["fanout"] for sc in scs} == set(range(1, 9))
    assert {sc.slots for sc in scs} >= set(range(9, 17))
    assert {sc.topology for sc in scs} == set(E.TOPOLOGIES)


# ---- scheduler switches ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("switches", [("SERFSIM_NO_SKIP",), ("SERFSIM_NO_JUMP",), ("SERFSIM_NO_SKIP", "SERFSIM_NO_JUMP")])
def test_scheduler_switches_change_nothing(switches, monkeypatch):
    """DESIGN §5: skipping idle tiles / ticks and jumping over sleeping stretches changes no row, record or clock."""
    scs = [E.crash_study(5000, random_regular_graph(5000, 12, 8), fanout=4)] + [E.envelope_fuzz(s) for s in range(4)]
    base = [P.run_against_oracle(emu_sim, sc, traces=(0,)) for sc in scs]
    for k in switches:
        monkeypatch.setenv(k, "1")
    for sc, out in zip(scs, base):
        P.assert_same(P.run_against_oracle(emu_sim, sc, traces=(0,)), out, with_hash=True, what=sc.name)


# ---- sharded: shards that do and do not have a uniform degree ---------------------------------------------------
def mixed_graph(n, world, seed=2):
    """Shard 0 has uniform degree 8, shard 1 irregular degrees, shard 2 (world 3) uniform degree 5: each shard decides for itself
    whether its row offsets are arithmetic, and shards after the first start at an edge offset e0 ≠ 0."""
    shard = (n + world - 1) // world
    rng = np.random.Generator(np.random.Philox(seed))
    irr = E.irregular_graph(n, seed + 1, hubs=1, hub_degree=(300, 600))[0]
    deg = np.diff(irr.astype(np.int64))
    deg[:shard] = 8
    if world > 2:
        deg[2 * shard:] = 5
    col = rng.integers(0, n - 1, size=int(deg.sum()), dtype=np.int64)
    src = np.repeat(np.arange(n), deg)
    col += col >= src
    rp = np.zeros(n + 1, np.uint64)
    rp[1:] = np.cumsum(deg)
    return rp, col.astype(np.uint32), shard


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_mixed_uniform_and_irregular_shards(world):
    from serf_b200.scenarios import Scenario
    from serf_b200.sim import Op
    n = 3001
    rp, col, shard = mixed_graph(n, world)
    deg = np.diff(rp.astype(np.int64))
    assert (deg[:shard] == 8).all() and np.unique(deg[shard:2 * shard]).size > 2
    sc = Scenario(f"mixed_{world}", n, 2, (rp, col), [3, shard + 7], [(0, Op.LEAVE, 3, 0), (0, Op.FAIL, shard + 7, 0)],
                  dict(fanout=4, seed=3, suspicion_mult=2, suspicion_max_timeout_mult=2, probe_interval_ticks=2), max_ticks=120)
    P.run_against_oracle(emu_sim, sc, world=world)


# ---- ABI limits --------------------------------------------------------------------------------------------------
def _star(n, hub_degree):
    deg = np.ones(n, np.int64)
    deg[1] = hub_degree
    rp = np.zeros(n + 1, np.uint64)
    rp[1:] = np.cumsum(deg)
    col = (np.arange(int(deg.sum())) % (n - 1) + 2) % n
    return rp, col.astype(np.uint32)


def test_degree_limit():
    g = emu_sim(300, 1)
    g.set_topology(*_star(300, 65535))
    with pytest.raises(SerfsimError) as e:
        emu_sim(300, 1).set_topology(*_star(300, 65536))
    assert e.value.code == -1 and "65535" in str(e.value)
    g.set_subjects(np.array([1], np.uint32))
    g.leave(1)
    assert g.run_until_converged(500)[1]


@pytest.mark.parametrize("kw", [dict(fanout=0), dict(fanout=9), dict(slots=0), dict(slots=17)])
def test_fanout_and_slot_limits_are_rejected(kw):
    slots = kw.pop("slots", 1)
    with pytest.raises(SerfsimError) as e:
        emu_sim(100, slots, **kw)
    assert e.value.code == -1


def test_fanout8_slots16_accepted_and_exact():
    n = 600
    rng = np.random.Generator(np.random.Philox(3))
    subjects = rng.choice(n, 16, replace=False)
    from serf_b200.scenarios import Scenario
    from serf_b200.sim import Op
    ops = [(0, Op.LEAVE, int(s), 0) for s in subjects[:8]] + [(1, Op.FAIL, int(s), 0) for s in subjects[8:]]
    sc = Scenario("f8_r16", n, 16, E.irregular_graph(n, 5, hubs=1), subjects, ops,
                  dict(fanout=8, seed=9, suspicion_mult=2, suspicion_max_timeout_mult=2, probe_interval_ticks=1), max_ticks=150)
    P.run_against_oracle(emu_sim, sc)
