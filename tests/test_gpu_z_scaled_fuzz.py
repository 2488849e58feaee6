"""Every feature at once at multi-tile scale on the device, against the oracle: the seeds of tests/test_emu_scaled_fuzz.py at
20 K – 200 K nodes (scaled_fuzz_lib.scaled_fuzz), in trace mode (general kernel, per-tick hash) and in production mode (per-view
passes, compaction, skipped and jumped ticks) — records of every slot, clocks, every getter, every trace row, stats, the state hash,
user-event records / stats / clocks / seen vectors, anomaly flags and injector stats.

Only a multi-CTA launch on feature-rich traffic can show a race or an ordering mistake in the dedup peek before RED.MAX, the hot-tile
marks of sparse ticks, tile_due / node_due, the last-CTA ticket and sleep verdict, the carry words between passes, the per-view kind
counters or the scheduler's jump rule.  A subset of the seeds runs again under every run-time switch (SERFSIM_SV 0 / 2,
SERFSIM_COMPACT=0, SERFSIM_AHEAD 0 / 2, SERFSIM_DEDUP=0, SERFSIM_NO_SKIP, SERFSIM_NO_JUMP, SERFSIM_CHUNK 3–7, SERFSIM_TMA=1 on the
single-slot seeds) and under SERFSIM_GRIDMUL=1 (several tiles per CTA).  The paths reached are derived from the
product's getters (scaled_fuzz_lib.reach) and asserted: a parity test that never reached them would prove little."""
import functools

import numpy as np
import pytest

import envelope_lib as E
import parity_lib as P
import scaled_fuzz_lib as S
from oracle_lib import oracle_sim, oracle_sim_threaded
from serf_b200 import GossipSim

pytestmark = pytest.mark.gpu

SEEDS = list(range(10))
MATRIX_SEEDS = [0, 2, 4, 5, 7, 9]


def size(device_n, emu_n):
    """The host build of the kernels (dry run of this file) runs the same seeds at sizes a fiber scheduler finishes."""
    return emu_n if E.ON_EMU else device_n


def scenario(seed):
    return S.scaled_fuzz(seed, n=size(None, 4000 + (seed * 7919) % 6000))


@functools.lru_cache(None)
def oracle(seed):
    """One oracle run (trace = 1) per seed, shared by every mode."""
    sc = scenario(seed)
    o = sc.build(oracle_sim_threaded if sc.n >= 100_000 else oracle_sim, trace=1)
    return sc, P.outputs(o, sc, o.run_until_converged(sc.max_ticks))


def run(sc, trace):
    g = sc.build(GossipSim, trace=trace)
    out = E.product_run(g, sc)
    g.close()
    return out


@functools.lru_cache(None)
def production(seed):
    sc, ref = oracle(seed)
    got = run(sc, 0)
    P.assert_same(got["out"], ref, with_hash=False, what=f"{sc.name} trace=0")
    return got


@pytest.mark.parametrize("seed", SEEDS)
def test_scaled_fuzz(seed):
    sc, ref = oracle(seed)
    assert sc.n % E.TILE != 0
    P.assert_same(run(sc, 1)["out"], ref, with_hash=True, what=f"{sc.name} trace=1")
    production(seed)


def test_device_reach():
    """The production runs reached per-view passes, compacted walks under another view's saturation, unread planes, sparse and dense
    ticks; and the host jumped over sleeping stretches (fewer launches than the same run under SERFSIM_NO_JUMP=1)."""
    reach = {s: S.reach(production(s), oracle(s)[0]) for s in SEEDS}
    for s, r in reach.items():
        print(f"\n{oracle(s)[0].name}: {r}", end="")
    print()
    hits = {k: sum(1 for r in reach.values() if r[k]) for k in ("pass_ticks", "compacted_under_other", "unread_plane", "sparse", "dense")}
    need = dict(pass_ticks=4, compacted_under_other=2, unread_plane=3, sparse=8, dense=8)
    assert all(hits[k] >= v for k, v in need.items()), (hits, need)


def test_jumps_launch_fewer_kernels(monkeypatch):
    jumped = 0
    for seed in MATRIX_SEEDS:
        sc, ref = oracle(seed)
        base = production(seed)
        monkeypatch.setenv("SERFSIM_NO_JUMP", "1")
        nj = run(sc, 0)
        monkeypatch.delenv("SERFSIM_NO_JUMP")
        P.assert_same(nj["out"], ref, with_hash=False, what=f"{sc.name} NO_JUMP")
        assert base["launches"] <= nj["launches"], (sc.name, base["launches"], nj["launches"])
        jumped += base["launches"] < nj["launches"]
    assert jumped >= 2, jumped


MODES = [dict(SERFSIM_SV="0"), dict(SERFSIM_SV="2"), dict(SERFSIM_COMPACT="0"), dict(SERFSIM_AHEAD="0"), dict(SERFSIM_AHEAD="2"),
         dict(SERFSIM_DEDUP="0"), dict(SERFSIM_NO_SKIP="1"), dict(SERFSIM_CHUNK="chunk")]


@pytest.mark.parametrize("mode", MODES, ids=lambda m: ",".join(f"{k[8:]}={v}" for k, v in m.items()))
def test_mode_matrix(mode, monkeypatch):
    """Production runs of the subset under one switch each; SERFSIM_CHUNK takes 3–7 ticks, a different chunk per seed."""
    for i, seed in enumerate(MATRIX_SEEDS):
        sc, ref = oracle(seed)
        for k, v in mode.items():
            monkeypatch.setenv(k, str(3 + i % 5) if v == "chunk" else v)
        got = run(sc, 0)
        P.assert_same(got["out"], ref, with_hash=False, what=f"{sc.name} {mode}")
        if mode.get("SERFSIM_SV") in ("0", "2"):
            assert not got["view_kinds"].any()                     # no tick ran as passes


def test_tma_on_single_slot_seeds(monkeypatch):
    scs = [s for s in range(40) if scenario(s).slots == 1][:2]
    assert len(scs) == 2
    monkeypatch.setenv("SERFSIM_TMA", "1")
    for seed in scs:
        sc, ref = oracle(seed)
        for trace in (1, 0):
            P.assert_same(run(sc, trace)["out"], ref, with_hash=bool(trace), what=f"{sc.name} TMA trace={trace}")


def test_several_tiles_per_cta(capfd):
    """SERFSIM_GRIDMUL=1: one wave of CTAs instead of two.  The multi-slot kernel runs one CTA per SM, so above
    132 · 256 nodes each of its CTAs owns several tiles — the multi-tile compaction groups of host-operation and reaper ticks."""
    seeds = [s for s in SEEDS if scenario(s).slots > 1 and scenario(s).n > size(40_000, 0)][:3]
    assert len(seeds) == 3
    res = E.run_jobs([dict(sc=oracle(s)[0], trace=t) for s in seeds for t in (1, 0)], capfd, {"SERFSIM_GRIDMUL": "1"})
    for i, got in enumerate(res):
        sc, ref = oracle(seeds[i // 2])
        P.assert_same(got["out"], ref, with_hash=i % 2 == 0, what=f"{sc.name} GRIDMUL=1")
        assert E.tiles_per_cta(sc.n, got["kernel"][1]) > 1, (sc.name, got["kernel"])
