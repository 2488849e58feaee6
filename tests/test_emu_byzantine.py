"""Byzantine-injector kernel logic on the CPU: byz_kernel.cu (and the host code around it) compiled for the host by
tests/emu, against the oracle's definition — the comparisons of tests/test_gpu_z_byzantine.py at small sizes."""
import pytest

import parity_lib as P
from emu_lib import emu_sim
from oracle_lib import oracle_sim
from serf_b200 import scenarios


@pytest.mark.parametrize("seed", [1, 2])
def test_config4_shape_one_percent(seed):
    sc = scenarios.byzantine_injectors(5000, 16, 4, 0.01, seed=seed)
    out = P.run_against_oracle(emu_sim, sc)
    assert out["anomaly_flags"][sc.byzantine].mean() > 0.9


def test_heavy_injection_changes_the_trace():
    sc = scenarios.byzantine_injectors(3000, 16, 4, 0.2, seed=3)
    out = P.run_against_oracle(emu_sim, sc)
    honest = scenarios.byzantine_injectors(3000, 16, 4, 0.2, seed=3)
    honest.byzantine = None
    h = honest.build(oracle_sim, trace=1)
    h.run_until_converged(honest.max_ticks)
    assert out["stats"] != h.stats()                      # the stale copies did change the honest dynamics in this run


def test_single_slot_no_probing():
    P.run_against_oracle(emu_sim, scenarios.byzantine_injectors(3000, 12, 3, 0.05, seed=2, churn=False, slots=1))


def test_delta_variants():
    P.run_against_oracle(emu_sim, scenarios.byzantine_injectors(2000, 12, 3, 0.05, delta=0, seed=2, churn=False, slots=1))
    P.run_against_oracle(emu_sim, scenarios.byzantine_injectors(2000, 12, 3, 0.05, delta=5, seed=2))


def test_injectors_and_user_events_together():
    sc = scenarios.byzantine_injectors(2500, 16, 4, 0.02, seed=6)
    ue = scenarios.user_event_storm(2500, 16, 4, seed=6, n_events=3)
    sc.user_events = ue.user_events
    sc.ops += [op for op in ue.ops if (op[0], op[2]) not in {(o[0], o[2]) for o in sc.ops}]
    P.run_against_oracle(emu_sim, sc)


@pytest.mark.parametrize("pp", [6, 15])
def test_injectors_with_push_pull_rounds(pp):
    """Verdicts of a tick are taken before that tick's push-pull round, on the device as in the oracle."""
    P.run_against_oracle(emu_sim, scenarios.byzantine_injectors(2500, 12, 3, 0.05, seed=5), push_pull_interval_ticks=pp)
