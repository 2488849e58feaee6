"""Device parity of the multi-slot kernel's alternative paths against the oracle: requests one tile ahead (SERFSIM_AHEAD: off / forced in
every tick) and the single-view dispatch (SERFSIM_SV: off / dual launch / check mode, where the general kernel runs alone and error 4 is
raised if a view outside a one-element set of views with business turns out to have business) — production mode (trace = 0) and trace
mode, a crash + leave study with LAN-like timers, multi-phase sequences (converge → crash → continue → rejoin), fuzz scenarios."""
import pytest

import parity_lib as P
from oracle_lib import oracle_sim
from serf_b200 import GossipSim, scenarios
from serf_b200.sim import Op

pytestmark = pytest.mark.gpu


MODES = [dict(SERFSIM_SV="0", SERFSIM_AHEAD="0"), dict(SERFSIM_SV="1", SERFSIM_AHEAD="2"), dict(SERFSIM_SV="2", SERFSIM_AHEAD="1"),
         dict(SERFSIM_SV="1", SERFSIM_AHEAD="2", SERFSIM_COMPACT="0")]


@pytest.mark.parametrize("mode", MODES, ids=lambda m: ",".join(f"{k[8:]}={v}" for k, v in m.items()))
def test_crash_and_leave_study(monkeypatch, mode):
    for k, v in mode.items():
        monkeypatch.setenv(k, v)
    for sc in (scenarios.dissemination_storm(200_000, 16, 4, slots=2, seed=3, with_fail=True), scenarios.dissemination_storm(60_000, 12, 3, slots=3, seed=5, with_fail=True)):
        P.run_against_oracle(GossipSim, sc, traces=(0, 1))


@pytest.mark.parametrize("mode", MODES[1:3], ids=lambda m: ",".join(f"{k[8:]}={v}" for k, v in m.items()))
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_multi_phase(monkeypatch, mode, seed):
    for k, v in mode.items():
        monkeypatch.setenv(k, v)
    monkeypatch.setenv("SERFSIM_CHUNK", "5")
    sc = scenarios.random_graph_leave(40_000, 12, 4, seed=seed, slots=3, graph_seed=seed + 30)
    cfg = dict(suspicion_mult=2, suspicion_max_timeout_mult=2, probe_interval_ticks=2)
    g, o = sc.build(GossipSim, trace=0, **cfg), sc.build(oracle_sim, trace=1, **cfg)
    assert g.run_until_converged(sc.max_ticks) == o.run_until_converged(sc.max_ticks)
    for sim in (g, o):
        sim.inject(sim.stats()["tick"], Op.FAIL, int(sc.subjects[1]), 0)           # from here on exactly one subject has ever been down
    tg, to = g.run_until_converged(5000), o.run_until_converged(5000)
    P.assert_same(P.outputs(g, sc, tg), P.outputs(o, sc, to), with_hash=False)
    for sim in (g, o):
        t = sim.stats()["tick"]
        sim.inject(t, Op.REJOIN, int(sc.subjects[1]), 0)
        sim.inject(t + 2, Op.FORCE_LEAVE, 11, 2)
    tg, to = g.run_until_converged(5000), o.run_until_converged(5000)
    P.assert_same(P.outputs(g, sc, tg), P.outputs(o, sc, to), with_hash=False)
    for sim in (g, o):
        sim.inject(sim.stats()["tick"] + 1, Op.FAIL, int(sc.subjects[2]), 0)       # a second subject goes down: the dispatch switches itself off
    tg, to = g.run_until_converged(5000), o.run_until_converged(5000)
    P.assert_same(P.outputs(g, sc, tg), P.outputs(o, sc, to), with_hash=False)


@pytest.mark.parametrize("mode", MODES[1:3], ids=lambda m: ",".join(f"{k[8:]}={v}" for k, v in m.items()))
def test_fuzz(monkeypatch, mode):
    for k, v in mode.items():
        monkeypatch.setenv(k, v)
    for seed in range(8):
        P.run_against_oracle(GossipSim, scenarios.fuzz(seed), traces=(0,))
