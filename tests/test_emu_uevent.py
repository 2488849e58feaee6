"""User-event kernel logic on the CPU: uevent_kernel.cu (and the host code around it) compiled for the host by
tests/emu, against the oracle's literal ring-buffer model — the comparisons of tests/test_gpu_z_uevent.py at sizes a
fiber scheduler finishes in seconds."""
import pytest

import parity_lib as P
from emu_lib import emu_sim
from oracle_lib import oracle_sim
from serf_b200 import scenarios
from serf_b200.sim import SerfsimError


@pytest.mark.parametrize("seed", [1, 2])
def test_user_event_storm(seed):
    out = P.run_against_oracle(emu_sim, scenarios.user_event_storm(4000, 16, 3, seed=seed, n_events=4, spacing=3))
    assert out["user_event_stats"]["event_queue"] == 0


def test_user_events_with_churn_and_leave():
    P.run_against_oracle(emu_sim, scenarios.user_event_storm(3000, 12, 3, seed=4, n_events=6, spacing=1, churn=60, with_leave=True))


def test_aliased_events():
    out = P.run_against_oracle(emu_sim, scenarios.user_event_storm(2500, 12, 3, seed=5, n_events=3, spacing=2, alias=True))
    assert ((out["user_event_seen"][0] + out["user_event_seen"][1]) == 1).all()


@pytest.mark.parametrize("fanout,events", [(1, 2), (4, 8), (8, 3)])
def test_fanouts_and_event_counts(fanout, events):
    P.run_against_oracle(emu_sim, scenarios.user_event_storm(1500, 10, fanout, seed=7, n_events=events, spacing=1, churn=20))


def test_user_events_with_failure_detection():
    sc = scenarios.user_event_storm(2500, 16, 3, seed=8, n_events=4, spacing=4)
    sc.ops.append((2, scenarios.Op.FAIL, 0, 0))
    P.run_against_oracle(emu_sim, sc, suspicion_mult=2, suspicion_max_timeout_mult=2, probe_interval_ticks=2)


def test_reset_clears_event_state():
    sc = scenarios.user_event_storm(1500, 12, 3, seed=2, n_events=3)
    g = sc.build(emu_sim, trace=1)
    g.run_until_converged(sc.max_ticks)
    h1, st1 = g.state_hash(), g.user_event_stats()
    g.reset(sc.cfg["seed"])
    assert g.user_event_stats()["delivered"] == 0 and (g.user_event_seen(0) == 0).all()
    sc.schedule(g)
    g.run_until_converged(sc.max_ticks)
    assert g.state_hash() == h1 and g.user_event_stats() == st1


def test_host_validation():
    sc = scenarios.user_event_storm(300, 8, 3, seed=1, n_events=2)
    g = sc.build(emu_sim)
    with pytest.raises(SerfsimError):
        g.user_event(5, 0, tick=9)                 # a tracked event fires once
    with pytest.raises(SerfsimError):
        g.user_event(5, 2, tick=9)                 # only 2 tracked events
    with pytest.raises(SerfsimError):
        g.set_user_events([1])                     # operations are already scheduled


@pytest.mark.parametrize("pp", [5, 13])
def test_user_events_with_push_pull_rounds(pp):
    """retransmit_mult 1 leaves the gossip of the events incomplete; push-pull rounds replay the partner's event ring
    (delegate.rs:539-552) and witness its event clock until everybody has everything."""
    sc = scenarios.user_event_storm(2500, 8, 2, seed=6, n_events=5, spacing=2, churn=30, with_leave=True)
    st = P.run_against_oracle(emu_sim, sc, push_pull_interval_ticks=pp, retransmit_mult=1)["user_event_stats"]
    gossip_only = scenarios.user_event_storm(2500, 8, 2, seed=6, n_events=5, spacing=2, churn=30, with_leave=True).build(oracle_sim, trace=1, retransmit_mult=1)
    gossip_only.run_until_converged(sc.max_ticks)
    assert st["delivered"] > gossip_only.user_event_stats()["delivered"]        # the rounds did deliver events gossip had missed
