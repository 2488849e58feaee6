"""Every feature at once at multi-tile scale on the host build of the kernels (tests/emu), against the oracle.

scaled_fuzz_lib.scaled_fuzz draws scenarios with every operation kind (prune, rejoin, user events with aliases), the reaper erasing
members mid-run, push-pull rounds, injectors, both timer profiles, and operations timed into every tick regime.  The committed seeds
run here at 6 K – 24 K nodes (24 – 94 tiles) in trace mode (general kernel, per-tick hash) and in production mode (per-view passes,
compaction, skipped and jumped ticks); tests/test_gpu_z_scaled_fuzz.py runs the same seeds at 20 K – 200 K nodes on the device.

A parity test proves little about paths the scenarios never reach, so the coverage probes of the host build (SFS_PROBE) are summed
over the production runs of the campaign and each targeted path must be reached by several scenarios:
 1 / 2   compaction groups of several tiles / with more than one dense pass     22  REDs the delivered-word peek skipped
 3 / 17  ticks skipped on the device / jumped over by the host                  23  passes on the whole-tick counters (fallback)
 4 / 20  tiles woken by the timer wheel / their nodes whose node_due lies later 24  compacted walk under another view's saturation
 21      per-view pass CTAs that ran                                            25  a plane left unread that another view sends
 26      per-delivery tile marks of sparse ticks                               27  reaper erases      28  push-pull record changes
"""
import ctypes as C
import functools

import pytest

import envelope_lib as E
import parity_lib as P
import scaled_fuzz_lib as S
from emu_lib import emu_sim, lib
from oracle_lib import oracle_sim

SEEDS = list(range(12))
PROBES = {1: "multi-tile compaction group", 2: "group > 256 active", 3: "skipped ticks", 17: "jumped ticks", 4: "timer-wheel tiles",
          20: "node_due later", 21: "per-view pass CTAs", 22: "dedup-skipped REDs", 23: "pass whole-tick fallback",
          24: "compacted walk under other view's saturation", 25: "plane left unread", 26: "sparse-tick tile marks", 27: "reaper erases",
          28: "push-pull record changes"}


def host_n(seed):
    """6 K – 24 K nodes: at least 23 tiles, spread over the 4 CTAs of the host build's default grid."""
    return 6000 + (seed * 7919) % 18000


def _probes():
    L = lib()
    L.emu_probe.restype = C.c_ulong
    return L


@functools.lru_cache(None)
def oracle_run(seed):
    sc = S.scaled_fuzz(seed, n=host_n(seed))
    o = sc.build(oracle_sim, trace=1)
    return sc, P.outputs(o, sc, o.run_until_converged(sc.max_ticks))


@functools.lru_cache(None)
def production_run(seed):
    """The host build in production mode (trace = 0), checked against the oracle; returns (outputs, the run's probe counts)."""
    sc, ref = oracle_run(seed)
    L = _probes()
    L.emu_probe_reset()
    got = E.product_run(sc.build(emu_sim, trace=0), sc)
    probes = {i: int(L.emu_probe(i)) for i in PROBES}
    P.assert_same(got["out"], ref, with_hash=False, what=f"{sc.name} trace=0")
    return got, probes


@pytest.mark.parametrize("seed", SEEDS)
def test_scaled_fuzz(seed):
    sc, ref = oracle_run(seed)
    assert sc.n % E.TILE != 0 and sc.n >= 16 * E.TILE
    g = sc.build(emu_sim, trace=1)
    P.assert_same(P.outputs(g, sc, g.run_until_converged(sc.max_ticks)), ref, with_hash=True, what=f"{sc.name} trace=1")
    production_run(seed)


def test_campaign_reaches_the_production_paths():
    runs = {s: production_run(s) for s in SEEDS}
    hits = {i: sum(1 for _, p in runs.values() if p[i] > 0) for i in PROBES}
    print(f"\nscaled_fuzz seeds {SEEDS[0]}–{SEEDS[-1]} on the host build, trace = 0: probe, total count, scenarios that hit it")
    for i, name in PROBES.items():
        print(f"  {i:2d} {name:46s} {sum(p[i] for _, p in runs.values()):>12d}  {hits[i]:2d} of {len(SEEDS)}")
    reach = {s: S.reach(got, oracle_run(s)[0]) for s, (got, _) in runs.items()}
    for k in ("pass_ticks", "compacted_under_other", "unread_plane", "sparse", "dense"):
        print(f"  getters: {k:24s} {sum(r[k] for r in reach.values()):>6d} ticks, {sum(1 for r in reach.values() if r[k]):2d} of {len(SEEDS)}")
    need = {1: 8, 2: 6, 4: 6, 20: 6, 21: 5, 22: 10, 23: 4, 24: 3, 25: 4, 26: 5, 27: 6, 28: 6}
    short = {PROBES[i]: (hits[i], k) for i, k in need.items() if hits[i] < k}
    assert not short, f"paths reached by too few scenarios (hits, needed): {short}"
    skipped_or_jumped = sum(1 for _, p in runs.values() if p[3] + p[17] > 0)
    assert skipped_or_jumped >= 4, skipped_or_jumped
    # the getters the device test derives its reach from agree with the probes
    for s, (got, p) in runs.items():
        assert not reach[s]["pass_ticks"] or p[21] > 0, (s, reach[s], p[21])
        assert not reach[s]["compacted_under_other"] or p[24] > 0, (s, reach[s], p[24])
        assert not reach[s]["unread_plane"] or p[25] > 0, (s, reach[s], p[25])


def test_random_schedule_and_grid_change_nothing():
    """Another lane / CTA order (a fresh process: the host build reads it once) and another grid give the same results bit for bit."""
    seed = 2
    sc, ref = oracle_run(seed)
    got = E.run_isolated([dict(sc=sc, trace=0)], {"SERFSIM_EMU_SCHED": "random:11", "SERFSIM_EMU_SMS": "3"})[0]
    P.assert_same(got["out"], ref, with_hash=False, what=f"{sc.name} random schedule")
    base, _ = production_run(seed)
    assert (got["view_kinds"] == base["view_kinds"]).all()
