"""Production mode (trace = 0: tile skipping, lazy loads, compaction) across converge → inject → continue sequences on
the device — the mirror of tests/test_emu_host.py::test_multi_phase_production_mode_rewind (ADVICE r1: the convergence
loop's rewind used to drop the watcher tiles' flags after an odd number of speculative ticks)."""
import pytest

import parity_lib as P
from oracle_lib import oracle_sim
from serf_b200 import GossipSim, scenarios
from serf_b200.sim import Op

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("seed", range(1, 9))
@pytest.mark.parametrize("chunk", ["4", "3"])
def test_multi_phase_production_mode(monkeypatch, seed, chunk):
    monkeypatch.setenv("SERFSIM_CHUNK", chunk)
    sc = scenarios.random_graph_leave(30_000, 12, 3, seed=seed, slots=2, graph_seed=seed + 20)
    cfg = dict(suspicion_mult=2, suspicion_max_timeout_mult=2, probe_interval_ticks=2)
    sc.ops = [(0, Op.JOIN, int(sc.subjects[0]), 0)]
    g, o = sc.build(GossipSim, trace=0, **cfg), sc.build(oracle_sim, trace=1, **cfg)
    assert g.run_until_converged(sc.max_ticks) == o.run_until_converged(sc.max_ticks)
    for sim in (g, o):
        sim.inject(sim.stats()["tick"], Op.FAIL, int(sc.subjects[1]), 0)
    tg, to = g.run_until_converged(5000), o.run_until_converged(5000)
    P.assert_same(P.outputs(g, sc, tg), P.outputs(o, sc, to), with_hash=False)
    for sim in (g, o):
        t = sim.stats()["tick"]
        sim.inject(t, Op.REJOIN, int(sc.subjects[1]), 0)
        sim.inject(t + 3, Op.FORCE_LEAVE, 7, 0)
    tg, to = g.run_until_converged(5000), o.run_until_converged(5000)
    P.assert_same(P.outputs(g, sc, tg), P.outputs(o, sc, to), with_hash=False)
