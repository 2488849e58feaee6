"""GPU parity for user-event dissemination (SURVEY §8f row 3): the CUDA path through the C ABI against the oracle's
literal ring-buffer model, bit for bit — 16-byte event records, event clocks, stamped Lamport times, every trace row
(user-event deliveries are part of edge_updates / messages / changed / pending / hash), counters and the state hash.
"""
import pytest

import parity_lib as P
from serf_b200 import GossipSim, scenarios

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_user_event_storm_100k(seed):
    out = P.run_against_oracle(GossipSim, scenarios.user_event_storm(100_000, 16, 3, seed=seed, n_events=4, spacing=3))
    assert out["user_event_stats"]["event_queue"] == 0


def test_user_events_with_churn_and_leave():
    P.run_against_oracle(GossipSim, scenarios.user_event_storm(40_000, 16, 3, seed=4, n_events=6, spacing=1, churn=300, with_leave=True))


def test_aliased_events():
    out = P.run_against_oracle(GossipSim, scenarios.user_event_storm(30_000, 12, 3, seed=5, n_events=3, spacing=2, alias=True))
    both = out["user_event_seen"][0] + out["user_event_seen"][1]
    assert (both <= 1).all() and (both == 1).mean() > 0.999           # never both; a random digraph may strand a node or two with neither


@pytest.mark.parametrize("fanout,events", [(1, 2), (4, 8), (8, 3)])
def test_fanouts_and_event_counts(fanout, events):
    P.run_against_oracle(GossipSim, scenarios.user_event_storm(20_000, 10, fanout, seed=7, n_events=events, spacing=1, churn=50))


def test_user_events_with_failure_detection():
    """Probing on, a tracked subject down: the membership kernel runs its watcher path while events are in flight."""
    sc = scenarios.user_event_storm(20_000, 16, 3, seed=8, n_events=4, spacing=4, with_leave=False)
    sc.ops.append((2, scenarios.Op.FAIL, 0, 0))
    P.run_against_oracle(GossipSim, sc, suspicion_mult=2, suspicion_max_timeout_mult=2, probe_interval_ticks=2)


def test_reset_clears_event_state():
    sc = scenarios.user_event_storm(5_000, 12, 3, seed=2, n_events=3)
    g = sc.build(GossipSim, trace=1)
    g.run_until_converged(sc.max_ticks)
    h1, st1 = g.state_hash(), g.user_event_stats()
    g.reset(sc.cfg["seed"])
    assert g.user_event_stats()["delivered"] == 0 and (g.user_event_seen(0) == 0).all()
    sc.schedule(g)
    g.run_until_converged(sc.max_ticks)
    assert g.state_hash() == h1 and g.user_event_stats() == st1


@pytest.mark.parametrize("pp", [5, 13])
def test_user_events_with_push_pull_rounds(pp):
    """retransmit_mult 1 leaves the gossip of the events incomplete; push-pull rounds replay the partner's event ring."""
    P.run_against_oracle(GossipSim, scenarios.user_event_storm(30_000, 8, 2, seed=6, n_events=5, spacing=2, churn=100, with_leave=True), push_pull_interval_ticks=pp, retransmit_mult=1)


@pytest.mark.parametrize("seed", range(12))
def test_fuzz_with_user_events_and_injectors(seed):
    """Every operation kind, reaper, probing, tracked user events (with aliases) and byzantine injectors at once."""
    sc = scenarios.fuzz_features(seed)
    sc.max_ticks = 1200
    P.run_against_oracle(GossipSim, sc)
