"""The configuration range of tests/test_config_envelope.py on the device, against the oracle: config_fuzz at small sizes and
at 10^4 / 10^5 ± 1 nodes, a k = 7 Lifeguard study with full confirmer sets, transmit budgets of 252 and 248 (the bench's shape)
through the single-slot kernels, whose per-CTA counters are packed into 16-bit halves, and the SERFSIM_E_OVERFLOW contract at
100 K nodes in production mode (idle-node skipping, sleeping views and the per-view passes are live there).

With SERFSIM_GPU_TESTS_ON_EMU=1 the same cases run on the host build of the kernels at smaller sizes (a dry run of this file).
"""
import numpy as np
import pytest

import config_lib as CL
import envelope_lib as E
import parity_lib as P
from oracle_lib import oracle_sim, oracle_sim_threaded
from serf_b200 import GossipSim, MlState, scenarios
from serf_b200.scenarios import Op, Scenario
from serf_b200.sim import random_regular_graph
from test_config_envelope import assert_overflow_at, overflow_scenario

pytestmark = pytest.mark.gpu


POPCOUNT = np.array([bin(i).count("1") for i in range(1 << 16)], dtype=np.int64)


def size(device_n, emu_n):
    return emu_n if E.ON_EMU else device_n


def device_sim(n, slots=1, **kw):
    return GossipSim(n, slots, **kw)


def check(jobs, capfd):
    """Run the jobs through the library and compare each with the oracle (trace = 1)."""
    res = E.run_jobs(jobs, capfd)
    oracles = {}
    for job, got in zip(jobs, res):
        sc = job["sc"]
        if id(sc) not in oracles:
            o = sc.build(oracle_sim_threaded if sc.n >= 100_000 else oracle_sim, trace=1, **job.get("cfg", {}))
            oracles[id(sc)] = P.outputs(o, sc, o.run_until_converged(sc.max_ticks))
            assert CL.max_ltime(o, sc.slots) < CL.LTIME_LIMIT, sc.name
        P.assert_same(got["out"], oracles[id(sc)], with_hash=bool(job["trace"]), what=f"{sc.name} trace={job['trace']}")
    return res


def test_config_fuzz_small(capfd):
    scs = [CL.config_fuzz(s) for s in range(40)]
    check([dict(sc=sc, trace=t) for sc in scs for t in (1, 0)], capfd)


LARGE = (9_999, 10_000, 10_001, 99_999, 100_000, 100_001)


@pytest.mark.parametrize("n", LARGE)
def test_config_fuzz_at_a_power_of_ten(n, capfd):
    """Drawn configs at 10^4 / 10^5 ± 1 nodes: the retransmit limit gains a digit and the node scale is exact at 10^k."""
    n = size(n, n // 100 + n % 10)
    sc = CL.config_fuzz(9_000 + n, n=n)
    sc.max_ticks = 200
    check([dict(sc=sc, trace=1), dict(sc=sc, trace=0)], capfd)


def test_lifeguard_k7_full_confirmer_sets():
    """suspicion_mult 9 (k = 7) and probing every tick, a crash at tick 0: 300 extra watchers point at the subject, so views collect
    all 8 confirmer buckets.  Every suspect view's deadline − the tick it became Suspect is the product's table entry for its
    confirmations; the run matches the oracle tick by tick."""
    n = size(50_000, 3_000)
    row_ptr, col = random_regular_graph(n, 16, 21)
    rng = np.random.Generator(np.random.Philox(3))
    col = col.copy()
    col[rng.choice(np.arange(10, n), size=300, replace=False) * 16] = 3
    cfg = dict(fanout=4, seed=9, suspicion_mult=9, suspicion_max_timeout_mult=10, probe_interval_ticks=1, gossip_interval_ms=7)
    table = CL.expected_suspicion_table(9, 10, 1, 7, n)
    assert len(table) == 8
    sc = Scenario("lifeguard_k7_device", n, 1, (row_ptr, col), [3], [(0, Op.FAIL, 3, 0)], cfg, max_ticks=table[0] + 40)
    for trace in (1, 0):
        g, o = sc.build(device_sim, trace=trace), sc.build(oracle_sim, trace=1)
        t0 = np.full(n, -1, dtype=np.int64)
        full = 0
        for _ in range(sc.max_ticks):
            g.step(1)
            o.step(1)
            t = g.stats()["tick"] - 1
            r = g.records(0)
            sus = (r["ml"] & 3) == MlState.SUSPECT
            t0[sus & (t0 < 0)] = t
            live = np.nonzero(sus & (r["deadline"] != 0))[0]
            c = POPCOUNT[r["conf_mask"][live]] - 1
            assert (r["deadline"][live].astype(np.int64) - t0[live] == np.asarray(table)[c]).all(), (trace, t)
            full += int((c == 7).sum())
            assert (r == o.records(0)).all(), (trace, t)
        assert full > 100, full                                    # 8-bit confirmer masks occurred
        assert ((g.records(0)["ml"] & 3) == MlState.DEAD).sum() > n // 2
        P.assert_same(P.outputs(g, sc, None), P.outputs(o, sc, None), with_hash=bool(trace))


def _budget_check(stats, limit, n):
    m = stats["messages"]
    assert m % limit == 0 and m // limit >= n - 1, (m, limit)           # every accepted entry sent exactly `limit` times


@pytest.mark.parametrize("mult,n", [(63, 5_000), (63, 9_999)])
def test_transmit_budget_252(mult, n, capfd):
    """retransmit_mult 63 at 1000–9999 nodes: a limit of 252 through the single-slot kernels (a leave study and a crash study)."""
    limit = CL.expected_retransmit_limit(mult, n)
    assert limit == 252
    topo = random_regular_graph(n, 16, 5)
    leave = E.leave_study(n, topo, fanout=4, seed=3, max_ticks=600)
    crash = E.crash_study(n, topo, fanout=4, seed=3, short_timers=True, max_ticks=600)
    for sc in (leave, crash):
        sc.cfg["retransmit_mult"] = mult
    res = check([dict(sc=sc, trace=t) for sc in (leave, crash) for t in (1, 0)], capfd)
    _budget_check(res[0]["out"]["stats"], limit, n)


def test_transmit_budget_248_at_the_bench_shape():
    """The bench's shape (10 M-node random graph of degree 16, fan-out 4, one leave) at retransmit_mult 31: a limit of 248."""
    n = size(10_000_000, 20_000)
    sc = scenarios.dissemination_storm(n, 16, 4, slots=1, seed=1)
    sc.cfg["retransmit_mult"] = 31
    limit = CL.expected_retransmit_limit(31, n)
    assert limit == (248 if n == 10_000_000 else 155)
    g = sc.build(device_sim, trace=0)
    tg = g.run_until_converged(sc.max_ticks)
    o = sc.build(oracle_sim_threaded, trace=0)
    got = P.outputs(g, sc, tg)
    P.assert_same(got, P.outputs(o, sc, o.run_until_converged(sc.max_ticks)), with_hash=False)
    _budget_check(got["stats"], limit, n - 16)


@pytest.mark.parametrize("slots", [1, 3])
def test_overflow_contract_at_100k_nodes(slots):
    """Production mode (trace 0) at 100 K nodes, one tick per call in lockstep with the oracle: every step before the first one
    after which the oracle holds a Lamport time ≥ LTIME_LIMIT succeeds and matches, that one fails with SERFSIM_E_OVERFLOW."""
    n = size(100_000, 2_000)
    assert_overflow_at(overflow_scenario(n=n, slots=slots, seed=5, horizon=200), 0, factory=device_sim)
    sc = overflow_scenario(n=n, slots=slots, init_clock=2, init_status_ltime=CL.INIT_LTIME_BOUND - 1, seed=6, horizon=200)
    assert_overflow_at(sc, 0, factory=device_sim)
