"""GPU parity for byzantine stale-record injectors (BASELINE configs[4]): CUDA path through the C ABI vs the oracle,
bit for bit — anomaly flags, injector counters, and everything the honest parity tests compare (records, clocks, every
trace row, state hash), with the per-tick hash on (trace = 1) and in production mode (trace = 0, tile skipping on).
The model is defined by the oracle (no reference semantics, SURVEY §7.4)."""
import pytest

import parity_lib as P
from serf_b200 import GossipSim, scenarios

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("seed", [1, 2])
def test_config4_shape_100k_one_percent(seed):
    sc = scenarios.byzantine_injectors(100_000, 16, 4, 0.01, seed=seed)
    out = P.run_against_oracle(GossipSim, sc)
    assert out["anomaly_flags"][sc.byzantine].mean() > 0.95


def test_heavy_injection_changes_the_trace():
    """20 % injectors: stale copies are accepted by lagging nodes and re-gossiped, so the honest trace itself differs
    from the injector-free run — and must still match the oracle."""
    P.run_against_oracle(GossipSim, scenarios.byzantine_injectors(30_000, 16, 4, 0.2, seed=3))


def test_single_slot_no_probing():
    P.run_against_oracle(GossipSim, scenarios.byzantine_injectors(40_000, 12, 3, 0.05, seed=2, churn=False, slots=1))


def test_delta_variants():
    P.run_against_oracle(GossipSim, scenarios.byzantine_injectors(20_000, 12, 3, 0.05, delta=0, seed=2, churn=False, slots=1))
    P.run_against_oracle(GossipSim, scenarios.byzantine_injectors(20_000, 12, 3, 0.05, delta=5, seed=2))


def test_injectors_and_user_events_together():
    sc = scenarios.byzantine_injectors(20_000, 16, 4, 0.02, seed=6)
    ue = scenarios.user_event_storm(20_000, 16, 4, seed=6, n_events=3)
    sc.user_events = ue.user_events
    sc.ops += [op for op in ue.ops if (op[0], op[2]) not in {(o[0], o[2]) for o in sc.ops}]
    P.run_against_oracle(GossipSim, sc)


@pytest.mark.parametrize("pp", [6, 15])
def test_injectors_with_push_pull_rounds(pp):
    """Verdicts of a tick are taken before that tick's push-pull round, on the device as in the oracle."""
    P.run_against_oracle(GossipSim, scenarios.byzantine_injectors(30_000, 12, 3, 0.05, seed=5), push_pull_interval_ticks=pp)
