"""Device parity at the edges of the ABI's input range, against the CPU oracle — the comparisons of tests/test_gpu_parity.py
(stats, every trace row with its hash when trace = 1, clocks, every slot's records and getters, state hash), in trace mode
and in production mode:

- CSR topologies whose out-degrees differ (row_ptr loaded, isolated nodes, hubs, self-loops, duplicate edges) on the
  direct-load kernel, the TMA pipeline and its barrier-synchronised form; a uniform graph forced through the general path;
- a tile's CSR span exactly at the 48 KB TMA stage (TMA selected) and one edge over (direct kernel selected);
- single-slot runs in which every CTA owns nine tiles or more, with a ragged last tile and CTAs the ceiling split leaves empty:
  the TMA pipeline's stage reuse across tiles, multi-tile compaction, the timer wheel's per-CTA scans;
- the scheduler switches SERFSIM_NO_SKIP / SERFSIM_NO_JUMP;
- fan-out 6–8 with 9–16 slots, run as per-view passes.

Every run reads its switches when its handle is created (envelope_lib.run_jobs), and reports the kernel and grid SERFSIM_VERBOSE
printed for it."""
import functools

import pytest

import envelope_lib as E
import parity_lib as P
from oracle_lib import oracle_sim, oracle_sim_threaded
from serf_b200 import GossipSim
from serf_b200.sim import random_regular_graph
from test_gpu_z_multislot_paths import MODES

pytestmark = pytest.mark.gpu

DIRECT, TMA = "tick_kernel", "tick_kernel_tma"
KERNELS = {"direct": ({}, DIRECT), "tma": ({"SERFSIM_TMA": "1"}, TMA), "tma_sync": ({"SERFSIM_TMA": "1", "SERFSIM_TMA_SYNC": "1"}, TMA)}


def size(device_n, emu_n):
    """The host build of the kernels (dry run of this file) runs the same cases at sizes a fiber scheduler finishes."""
    return emu_n if E.ON_EMU else device_n


_ORACLES = {}


def oracle(sc, cfg=None):
    """The outputs of the oracle's run of a scenario (trace = 1), kept for the other variants of the same test."""
    cfg = cfg or {}
    key = (id(sc), tuple(sorted(cfg.items())))
    if key not in _ORACLES:
        o = sc.build(oracle_sim_threaded if sc.n >= 100_000 else oracle_sim, trace=1, **cfg)
        _ORACLES[key] = (sc, P.outputs(o, sc, o.run_until_converged(sc.max_ticks)))          # (sc is kept alive: its id is the key)
    return _ORACLES[key][1]


def check(jobs, env, capfd, expect_kernel=None):
    """Run the jobs under the switches env and compare each with the oracle; returns the outputs."""
    res = E.run_jobs(jobs, capfd, env)
    for job, got in zip(jobs, res):
        sc = job["sc"]
        what = f"{sc.name} trace={job['trace']} {env}"
        P.assert_same(got["out"], oracle(sc, job.get("cfg", {})), with_hash=bool(job["trace"]), what=what)
        if expect_kernel:
            assert E.is_kernel(got["kernel"][0], expect_kernel), (what, got["kernel"])
    return res


def both(*scs, cfg=None):
    return [dict(sc=sc, trace=t, cfg=cfg or {}) for sc in scs for t in (1, 0)]


# ---- irregular CSR ---------------------------------------------------------------------------------------------
@functools.lru_cache(None)
def irregular_scenarios():
    n = size(100_000, 12_000)
    topo = E.irregular_graph(n, 3, hub_degree=(1000, 3000))
    assert E.max_tile_span_bytes(topo[0]) <= E.TMA_STAGE_BYTES
    fz = [E.envelope_fuzz(s, topology="irregular", slots=1) for s in range(16)]
    assert all(E.max_tile_span_bytes(sc.row_ptr) <= E.TMA_STAGE_BYTES for sc in fz)
    return (E.leave_study(n, topo, fanout=4), E.crash_study(n, E.irregular_graph(n, 4, self_loops=0.03, duplicates=0.05), fanout=3,
                                                            short_timers=True)), fz


@pytest.mark.parametrize("kernel", list(KERNELS))
def test_irregular_csr(kernel, capfd):
    env, name = KERNELS[kernel]
    studies, fz = irregular_scenarios()
    check(both(*studies) + both(*fz), env, capfd, name)


def test_uniform_graph_forced_through_general_path(capfd):
    n = size(100_000, 8000)
    sc = E.crash_study(n, random_regular_graph(n, 16, 9), fanout=4, short_timers=True)
    a = check(both(sc), {}, capfd)
    b = check(both(sc), {"SERFSIM_UDEG": "0"}, capfd)
    for x, y in zip(a, b):
        P.assert_same(y["out"], x["out"], with_hash=True, what="SERFSIM_UDEG=0")


# ---- TMA stage boundary ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("over", [0, 4], ids=["at_48k", "one_edge_over"])
def test_tma_stage_boundary(over, capfd):
    n = size(60_000, 4000)
    topo = E.tma_span_graph(n, E.TMA_STAGE_BYTES + over)
    assert E.max_tile_span_bytes(topo[0]) == E.TMA_STAGE_BYTES + (16 if over else 0)
    scs = (E.leave_study(n, topo, fanout=4), E.crash_study(n, topo, fanout=3, short_timers=True))
    check(both(*scs), {"SERFSIM_TMA": "1"}, capfd, DIRECT if over else TMA)


# ---- several tiles per CTA --------------------------------------------------------------------------------------------
TILES_PER_CTA = 9
MULTI = {"direct": ({"SERFSIM_GRIDMUL": "1"}, DIRECT, TILES_PER_CTA), "tma": ({"SERFSIM_GRIDMUL": "1", "SERFSIM_TMA": "1"}, TMA, TILES_PER_CTA),
         "tma_sync": ({"SERFSIM_GRIDMUL": "1", "SERFSIM_TMA": "1", "SERFSIM_TMA_SYNC": "1"}, TMA, TILES_PER_CTA),
         "minb5": ({"SERFSIM_GRIDMUL": "1", "SERFSIM_MINB": "5"}, DIRECT, 5)}


@functools.lru_cache(None)
def multi_tile_scenarios(g):
    """n from the direct kernel's printed grid g: T = 8·g + 1 tiles gives every busy CTA ⌈T / g⌉ = 9 tiles, leaves the CTAs
    past ⌈T / 9⌉ empty and the last busy one a single tile; the last tile holds 77 nodes."""
    tiles = (TILES_PER_CTA - 1) * g + 1
    n = (tiles - 1) * E.TILE + 77
    topo = random_regular_graph(n, 16, 7)
    return n, g, (E.leave_study(n, topo, fanout=4), E.crash_study(n, topo, fanout=4), E.crash_study(n, topo, fanout=3, short_timers=True))


@pytest.mark.parametrize("variant", list(MULTI))
def test_several_tiles_per_cta(variant, capfd):
    env, name, min_tiles = MULTI[variant]
    _, g = E.grid_for(GossipSim, 1 << 20, capfd, {"SERFSIM_GRIDMUL": "1"})
    n, g0, (leave, crash_lan, crash_short) = multi_tile_scenarios(g)
    jobs = both(leave) + [dict(sc=crash_lan, trace=0), dict(sc=crash_short, trace=0)]   # timer-wheel studies: production mode
    res = check(jobs, env, capfd, name)
    grid = res[0]["kernel"][1]
    per = E.tiles_per_cta(n, grid)
    print(f"{variant}: n {n}, grid {grid}, {per} tiles per CTA, {E.busy_ctas(n, grid)} CTAs with tiles")
    assert per >= min_tiles and n % E.TILE != 0
    if variant != "minb5":
        assert grid == g0 and E.busy_ctas(n, grid) < grid                 # trailing CTAs own no tile


# ---- scheduler switches -------------------------------------------------------------------------------------------------
@functools.lru_cache(None)
def switch_scenarios():
    n = size(100_000, 6000)
    crash = E.crash_study(n, E.irregular_graph(n, 8, hub_degree=(1000, 3000)), fanout=4)
    storm = E.crash_and_leave_study(size(60_000, 3000), random_regular_graph(size(60_000, 3000), 12, 5), fanout=3, slots=3)
    return [crash, storm], [E.envelope_fuzz(s) for s in range(8)]


_DEFAULT_SWITCH_RUNS = []


def default_switch_runs(capfd):
    """The scheduler-switch scenarios without a switch, run once for every test that compares with them."""
    if not _DEFAULT_SWITCH_RUNS:
        studies, fz = switch_scenarios()
        _DEFAULT_SWITCH_RUNS.extend(check(both(*studies) + [dict(sc=sc, trace=0) for sc in fz], {}, capfd))
    return _DEFAULT_SWITCH_RUNS


@pytest.mark.parametrize("env", [{"SERFSIM_NO_SKIP": "1"}, {"SERFSIM_NO_JUMP": "1"}, {"SERFSIM_NO_SKIP": "1", "SERFSIM_NO_JUMP": "1"}],
                         ids=["no_skip", "no_jump", "both"])
def test_scheduler_switches(env, capfd):
    studies, fz = switch_scenarios()
    res = check(both(*studies) + [dict(sc=sc, trace=0) for sc in fz], env, capfd)
    for got, base in zip(res, default_switch_runs(capfd)):
        P.assert_same(got["out"], base["out"], with_hash=True, what=str(env))


# ---- fan-out 6–8 × slots 9–16 -------------------------------------------------------------------------------------------
def wide_fuzz_seeds(k):
    out, s = [], 0
    while len(out) < k:
        sc = E.envelope_fuzz(s)
        if sc.cfg["fanout"] >= 6 and sc.slots >= 9:
            out.append(s)
        s += 1
    return out


@functools.lru_cache(None)
def wide_storm():
    n = size(200_000, 3000)
    return E.crash_and_leave_study(n, random_regular_graph(n, 16, 7), fanout=8, slots=12)


@pytest.mark.parametrize("mode", MODES, ids=lambda m: ",".join(f"{k[8:]}={v}" for k, v in m.items()))
def test_fanout8_slots12_storm(mode, capfd):
    sc = wide_storm()
    check(both(sc), mode, capfd)


def test_wide_fuzz(capfd):
    scs = [E.envelope_fuzz(s) for s in wide_fuzz_seeds(16)]
    assert {sc.cfg["fanout"] for sc in scs} == {6, 7, 8} and max(sc.slots for sc in scs) >= 15
    for mode in (MODES[0], MODES[1]):
        check([dict(sc=sc, trace=0) for sc in scs], mode, capfd)


def test_per_view_passes_ran(capfd):
    """Production run of the storm: every tick that runs as passes launches R kernels instead of one, so SERFSIM_SV=1 launches
    more kernels than SERFSIM_SV=0 — at least R − 1 = 11 more per tick for the ticks without a host operation."""
    sc = wide_storm()
    off = check([dict(sc=sc, trace=0)], {"SERFSIM_SV": "0"}, capfd)[0]
    on = check([dict(sc=sc, trace=0)], {"SERFSIM_SV": "1"}, capfd)[0]
    assert on["launches"] >= off["launches"] + (sc.slots - 1) * 5, (on["launches"], off["launches"])
