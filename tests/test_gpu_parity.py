"""GPU parity: the CUDA path (through the C ABI of libserfsim.so) against the CPU oracle, bit for bit.

Compared on the same seeded inputs: the raw 32-byte member records of every slot, the Lamport clock
of every node, the memberlist state/incarnation vectors, the convergence step count and EVERY field
of EVERY row of the per-tick trace (packets, edge-updates, messages, changed, pending, events,
suspects, state hash).  Integer work: the bar is exact equality.
"""
import numpy as np
import pytest

import parity_lib as P
from oracle_lib import oracle_sim
from serf_b200 import GossipSim, MemberStatus, scenarios

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_config0_full_mesh_256(seed):
    out = P.run_against_oracle(GossipSim, scenarios.full_mesh_leave(256, 3, seed))
    assert (out["member_status"][0][1:] == MemberStatus.LEFT).all()


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_config1_random_graph_100k(seed):
    out = P.run_against_oracle(GossipSim, scenarios.random_graph_leave(100_000, 16, 3, seed))
    assert (out["member_status"][0][1:] != MemberStatus.LEFT).sum() <= 3 and out["run"][0] < 100     # a random digraph may strand a node or two


def test_random_graph_multi_slot_fanout4():
    P.run_against_oracle(GossipSim, scenarios.random_graph_leave(60_000, 16, 4, seed=5, slots=4))


def test_failure_detection_random_graph():
    sc = scenarios.random_graph_fail(20_000, 16, 3, seed=2)
    out = P.run_against_oracle(GossipSim, sc, suspicion_mult=2, suspicion_max_timeout_mult=2, probe_interval_ticks=2)
    st = out["member_status"][0]
    assert (np.delete(st, 5) == MemberStatus.FAILED).all()


def test_failure_detection_lifeguard_confirmations():
    sc = scenarios.random_graph_fail(5_000, 24, 3, seed=4)
    P.run_against_oracle(GossipSim, sc, suspicion_mult=4, suspicion_max_timeout_mult=3, probe_interval_ticks=1, gossip_interval_ms=1000)


def test_config2_small_world_churn():
    sc = scenarios.small_world_churn(40_000, 16, 0.1, 0.05, slots=8, window=60, seed=3)
    P.run_against_oracle(GossipSim, sc, suspicion_mult=2, suspicion_max_timeout_mult=2, probe_interval_ticks=2)


@pytest.mark.parametrize("pp", [7, 16])
def test_push_pull_anti_entropy(pp):
    from serf_b200 import small_world_graph
    from serf_b200.scenarios import Scenario
    from serf_b200 import Op
    n = 20_000
    sc = Scenario("pushpull", n, 3, small_world_graph(n, 4, 0.05, 5), [7, 900, 15000],
                  [(0, Op.LEAVE, 7, 0), (3, Op.FAIL, 900, 0), (40, Op.FORCE_LEAVE, 11, 1), (5, Op.JOIN, 15000, 0)],
                  dict(fanout=2, retransmit_mult=1, seed=5, push_pull_interval_ticks=pp, probe_interval_ticks=2, suspicion_mult=2, suspicion_max_timeout_mult=2), max_ticks=3000)
    out = P.run_against_oracle(GossipSim, sc)
    assert (out["run"][0] + 1) % pp == 0


@pytest.mark.parametrize("seed", range(40))
def test_fuzz(seed):
    sc = scenarios.fuzz(seed)
    sc.max_ticks = 1500
    P.run_against_oracle(GossipSim, sc)


def test_remove_failed_node_prune_reference_scenario():
    """serf_remove_failed_node_prune (serf/base/tests/serf/remove.rs:95-165) and the same on a 20 K-node random graph: after the
    pruning force-leave no survivor lists the failed node any more."""
    for n in (3, 40, 20_000):
        out = P.run_against_oracle(GossipSim, scenarios.remove_failed_node_prune(n, at=40 if n < 1000 else 120))
        st = out["member_status"][0]
        assert (np.delete(st, 1) != MemberStatus.NONE).sum() <= (0 if n < 1000 else 3)


@pytest.mark.parametrize("seed", range(24))
def test_fuzz_prune(seed):
    sc = scenarios.fuzz_prune(seed)
    sc.max_ticks = 1500
    P.run_against_oracle(GossipSim, sc)


def test_stepwise_equals_batched_and_inject_midway():
    sc = scenarios.random_graph_leave(30_000, 16, 3, seed=8, slots=2)
    g, o = sc.build(GossipSim, trace=1), sc.build(oracle_sim, trace=1)
    for _ in range(6):
        g.step(1); o.step(1)
    g.remove_failed_node(77, 1, tick=9); o.remove_failed_node(77, 1, tick=9)
    g.step(7); o.step(7)
    P.assert_same(P.outputs(g, sc, None), P.outputs(o, sc, None), with_hash=True)
    tg, to = g.run_until_converged(500), o.run_until_converged(500)
    P.assert_same(P.outputs(g, sc, tg), P.outputs(o, sc, to), with_hash=True)


def test_reset_reproduces():
    sc = scenarios.random_graph_leave(50_000, 16, 3, seed=4)
    g = sc.build(GossipSim, trace=1)
    t1, _ = g.run_until_converged(500)
    h1, tr1 = g.state_hash(), g.tick_trace()
    g.reset(4)
    sc.schedule(g)
    t2, _ = g.run_until_converged(500)
    assert (t1, h1) == (t2, g.state_hash()) and (tr1 == g.tick_trace()).all()


def test_event_callback_reports_agreed_transitions():
    sc = scenarios.full_mesh_leave(256, 3, 1)
    g = sc.build(GossipSim)
    seen = []
    g.set_event_callback(lambda tick, ty, ids: seen.append((ty, tuple(ids))))
    g.run_until_converged(500)
    assert (1, (0,)) in seen            # MemberEventType::Leave for subject 0


def others_mask(status, subj):
    m = status != MemberStatus.LEFT
    m[subj] = False
    return m


# ---- full-size properties (no oracle at this size): BASELINE configs[3] shape on one GPU ----------
def test_full_size_10m_properties():
    sc = scenarios.dissemination_storm(10_000_000, 16, 4, slots=1, seed=1)
    g = sc.build(GossipSim, trace=1)
    ticks, ok = g.run_until_converged(400)
    assert ok
    st = g.stats()
    h1, tr1 = g.state_hash(), g.tick_trace()
    status = g.member_status(0)
    subj = int(sc.subjects[0])
    assert status[subj] == MemberStatus.LEAVING
    # a random digraph with Poisson(16) in-degree leaves O(1) of 10 M nodes unreachable (in-degree 0): they stay Alive
    others = np.delete(status, subj)
    missed = int((others != MemberStatus.LEFT).sum())
    assert missed <= 8 and set(np.unique(others)) <= {MemberStatus.ALIVE, MemberStatus.LEAVING, MemberStatus.LEFT, MemberStatus.FAILED}
    lt = g.status_ltime(0)
    assert ((lt == 2) | (others_mask(status, subj) & (lt == 1))).all()
    # every node that accepted an entry forwards it exactly retransmit_limit (32) times
    reached_intent = int((lt == 2).sum())
    reached_left = int((g.ml_state(0) == 3).sum())
    assert st["messages"] == 32 * (reached_intent + reached_left) and st["intent_queue"] == 0 and st["pending"] == 0
    assert tr1["hash"][-1] == h1
    # idempotence / determinism: same seed → same trace; extra ticks on a quiescent cluster change nothing
    g.step(3)
    assert g.state_hash() == h1
    g.reset(1); sc.schedule(g)
    t2, _ = g.run_until_converged(400)
    assert t2 == ticks and g.state_hash() == h1 and (g.tick_trace() == tr1).all()
